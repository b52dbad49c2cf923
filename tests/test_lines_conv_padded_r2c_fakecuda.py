"""CPU test of the non-dry host control flow of the real zero-padded 1-D convolve lines plans
(dfft_lines_plan_create_convolve_padded_r2c_1d), on the fake CUDA runtime of test_control_flow_fakecuda.py (device memory = host
memory, launches = counted no-ops): create -> 3 executes -> destroy in both precisions, with one launch per execute on the short
path and three on the long path between a start and an end event, a temporary of ceil(nlines / 2) * n complex elements on the long
path only (seen as the bytes the C allocator holds: the fake runtime's cudaMalloc is calloc) that destroy frees, nothing left
allocated, every execute-time rejection as its error code, and dfft_debug_launch_op refusing the four new records."""
import os
import subprocess
import sys
import textwrap

from test_control_flow_fakecuda import ROOT, fake_lib  # noqa: F401  (fixture)

WORKER = textwrap.dedent(r'''
    import ctypes, os, sys
    sys.path.insert(0, sys.argv[1])
    import distributedfft_b200.api as api
    api.LIB_PATH = sys.argv[2]
    api._lib = None
    import distributedfft_b200 as dfft
    L = dfft.lib()
    L.fakecuda_launches.restype = ctypes.c_longlong
    L.fakecuda_event_records.restype = ctypes.c_longlong
    L.fakecuda_live_allocations.restype = ctypes.c_longlong

    class MallInfo(ctypes.Structure):
        _fields_ = [(f, ctypes.c_size_t) for f in ("arena", "ordblks", "smblks", "hblks", "hblkhd", "usmblks", "fsmblks", "uordblks",
                                                   "fordblks", "keepcost")]
    libc = ctypes.CDLL(None)
    libc.mallinfo2.restype = MallInfo

    def held():
        m = libc.mallinfo2()
        return m.uordblks + m.hblkhd

    def alloc(nbytes):
        return dfft.fft_mpi_alloc_local_memory((nbytes + 15) // 16, dfft.ALLOC_DEV)

    SLACK = 1 << 20   # the plan object, its twiddle tables and the interpreter's own allocations

    def drive(precision, n, li, lo, nlines, flags=0):
        rsz = 4 if precision == dfft.FLOAT else 8
        a, b, m = alloc(nlines * li * rsz), alloc(nlines * lo * rsz), alloc((n // 2 + 1) * nlines * 2 * rsz)
        long_path = dfft.length_kind(n, precision) != 2
        temp = (nlines + 1) // 2 * n * 2 * rsz if long_path else 0
        h0 = held()
        plan = dfft.LinesConvolvePlan(one_d=(n, nlines), real_padded=(li, lo), precision=precision, flags=flags)
        grown = held() - h0
        assert temp <= grown < temp + SLACK, (n, nlines, temp, grown)
        l0, e0 = L.fakecuda_launches(), L.fakecuda_event_records()
        plan.execute(a, b, m, 1)
        plan.execute(a, b, m, nlines)
        if li == lo:
            plan.execute(a, a, m, 1)
        else:
            plan.execute(a, b, m, 1)
        plan.synchronize()
        assert L.fakecuda_event_records() - e0 == 6, L.fakecuda_event_records() - e0
        got = L.fakecuda_launches() - l0
        assert got == 3 * (3 if long_path else 1), (n, nlines, precision, got)
        plan.destroy()
        assert held() - h0 < SLACK, ("the temporary outlived the plan", n, held() - h0)
        for p in (a, b, m):
            L.dfft_free_local(p, dfft.ALLOC_DEV)

    for prec in (dfft.DOUBLE, dfft.FLOAT):
        for n in dfft.supported_lengths(prec):
            if n < 2:
                continue
            drive(prec, n, max(1, n // 2), max(1, n // 2), 5)
            drive(prec, n, n, 1, 3, dfft.SCALE_BACKWARD)
        for n, li, lo, nlines in ((8192, 4096, 4096, 64), (36, 20, 30, 7), (6144, 95, 6143, 16), (1 << 16, 1, 1 << 16, 9)):
            drive(prec, n, li, lo, nlines)
            drive(prec, n, li, li, nlines, dfft.SCALE_BACKWARD)

    def code(fn):
        try:
            fn()
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0])
        return 0

    def create(n, li, lo, nlines, precision=dfft.DOUBLE, flags=0):
        dfft.LinesConvolvePlan(one_d=(n, nlines), real_padded=(li, lo), precision=precision, flags=flags).destroy()

    assert code(lambda: create(64, 0, 8, 1)) == -1 and code(lambda: create(64, 8, 65, 1)) == -1
    assert code(lambda: create(8192, 1, 8192, 1 << 31)) == -3
    assert code(lambda: create(17, 1, 1, 1)) == -3 and code(lambda: create(1, 1, 1, 1)) == -3
    assert code(lambda: create(64, 8, 8, 1, flags=dfft.NO_FUSE)) == -1
    assert code(lambda: dfft.api._check(L.dfft_lines_plan_create_convolve_padded_r2c_1d(64, 8, 8, 1, dfft.DOUBLE, 0, None), "x")) == -1
    for n in (256, 8192):
        for prec in (dfft.DOUBLE, dfft.FLOAT):
            rsz = 4 if prec == dfft.FLOAT else 8
            csz = 2 * rsz
            nlines, li, lo = 7, n // 2, n // 2 + 3
            ib, ob, mb = nlines * li * rsz, nlines * lo * rsz, (n // 2 + 1) * csz
            a, b, m = alloc(ib + ob + 64), alloc(ob + 64), alloc(mb * nlines + 64)
            p = dfft.LinesConvolvePlan(one_d=(n, nlines), real_padded=(li, lo), precision=prec)
            assert code(lambda: p.execute(a, b, m, 1)) == 0
            assert code(lambda: p.execute(a, b, m, nlines)) == 0
            assert code(lambda: p.execute(a, a, m)) == -1                                   # in place needs in_len == out_len
            assert code(lambda: p.execute(a + ib - rsz, a, m)) == -1                       # partial overlaps of in and out
            assert code(lambda: p.execute(a, a + ib - rsz, m)) == -1
            assert code(lambda: p.execute(a, a + ib, m)) == 0                              # out right after in
            assert code(lambda: p.execute(a + ob, a, m)) == 0                              # in right after out
            mo = (ob + csz - 1) // csz * csz                                                # first complex-aligned byte past out
            assert code(lambda: p.execute(a, b, b + mo - csz)) == -1                       # multiplier overlaps out
            assert code(lambda: p.execute(a, b, b + mo)) == 0
            for mc in (0, 2, nlines + 1, -1):
                assert code(lambda: p.execute(a, b, m, mc)) == -1, mc
            assert code(lambda: p.execute(a + rsz // 2, b, m)) == -1                       # misaligned in / out / multiplier
            assert code(lambda: p.execute(a, b + rsz // 2, m)) == -1
            assert code(lambda: p.execute(a, b, m + rsz)) == -1
            assert code(lambda: p.execute(a + rsz, b + rsz, m)) == 0                       # real lines at an odd real offset
            assert code(lambda: dfft.api._check(L.dfft_lines_execute(p.handle, a, dfft.FORWARD), "x")) == -1
            p.synchronize(); p.destroy()
            q = dfft.LinesConvolvePlan(one_d=(n, nlines), real_padded=(li, li), precision=prec)
            assert code(lambda: q.execute(a, a, m)) == 0                                   # in place with in_len == out_len
            q.synchronize(); q.destroy()
            for x in (a, b, m):
                L.dfft_free_local(x, dfft.ALLOC_DEV)
    for rec in dfft.lines_conv_padded_1d_ops(64, 8, 8, 3, real=True) + dfft.lines_conv_padded_1d_ops(8192, 8, 8, 3, real=True):
        assert dfft.debug_launch_op(rec, dfft.DOUBLE) == -1, rec["op"]                     # lines-engine records are not replayed
    assert L.fakecuda_live_allocations() == 0, ("leak", L.fakecuda_live_allocations())
    print("real padded 1-D convolve lines fakecuda control flow ok")
''')


def test_real_padded_1d_convolve_lines_plans_run_to_completion_on_a_fake_runtime(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, DFFT_VERBOSE="1")
    for var in ("DFFT_NO_PLANE", "DFFT_FORCE_PLANE", "DFFT_GENERIC", "DFFT_VARIANT"):
        env.pop(var, None)
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "real padded 1-D convolve lines fakecuda control flow ok" in r.stdout
