"""CPU test of the non-dry host control flow of the batched 1-D convolve lines plans (dfft_lines_plan_create_convolve_1d /
_r2c_1d), on the fake CUDA runtime of test_control_flow_fakecuda.py (device memory = host memory, launches = counted no-ops):
create -> 3 executes -> destroy in both precisions with exactly one launch per execute and a start and end event around it,
nothing left allocated, and every execute-time rejection coming back as its error code."""
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

    def alloc(nbytes):
        return dfft.fft_mpi_alloc_local_memory((nbytes + 15) // 16, dfft.ALLOC_DEV)

    def drive(precision, n, nlines, real, flags=0):
        rsz = 4 if precision == dfft.FLOAT else 8
        io = n * nlines * (rsz if real else 2 * rsz)
        mline = n // 2 + 1 if real else n
        a, b, m = alloc(io), alloc(io), alloc(mline * nlines * 2 * rsz)
        plan = dfft.LinesConvolvePlan(one_d=(n, nlines), precision=precision, real=real, flags=flags)
        l0, e0 = L.fakecuda_launches(), L.fakecuda_event_records()
        plan.execute(a, b, m, 1)
        plan.execute(a, a, m, nlines)
        plan.execute(b, a, m, 1)
        plan.synchronize()
        assert L.fakecuda_event_records() - e0 == 6, L.fakecuda_event_records() - e0   # start and end event of every execute
        got = L.fakecuda_launches() - l0
        assert got == 3, (n, nlines, precision, real, got)                            # one launch per execute
        assert plan.stream
        plan.destroy()
        for p in (a, b, m):
            L.dfft_free_local(p, dfft.ALLOC_DEV)

    for prec in (dfft.DOUBLE, dfft.FLOAT):
        for n in dfft.supported_lengths(prec):
            drive(prec, n, 5, False)
            drive(prec, n, 5, True, dfft.SCALE_BACKWARD)
        for n, nlines in ((1024, 1), (256, 3), (768, 2), (1000, 7)):
            drive(prec, n, nlines, False, dfft.SCALE_BACKWARD)
            drive(prec, n, nlines, True)

    def code(fn):
        try:
            fn()
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0])
        return 0

    assert code(lambda: dfft.LinesConvolvePlan(one_d=(14, 1)).destroy()) == -3                # generic length
    assert code(lambda: dfft.LinesConvolvePlan(one_d=(8192, 1)).destroy()) == -3              # long line
    assert code(lambda: dfft.LinesConvolvePlan(one_d=(16, 1), flags=dfft.NO_FUSE).destroy()) == -1
    assert code(lambda: dfft.LinesConvolvePlan(one_d=(16, 1 << 31)).destroy()) == -3
    assert code(lambda: dfft.LinesConvolvePlan(one_d=(16, 1 << 31), real=True).destroy()) == -3
    assert code(lambda: dfft.LinesConvolvePlan(one_d=(1, 4), real=True).destroy()) == -3
    assert code(lambda: dfft.LinesConvolvePlan(one_d=(16, 1), precision=7).destroy()) == -1
    assert code(lambda: dfft.api._check(L.dfft_lines_plan_create_convolve_1d(16, 1, dfft.DOUBLE, 0, None), "x")) == -1
    assert code(lambda: dfft.api._check(L.dfft_lines_plan_create_convolve_r2c_1d(16, 1, dfft.DOUBLE, 0, None), "x")) == -1
    for bad in ({}, {"one_d": (16, 1), "two_d": (16, 16, 1)}, {"one_d": (16, 1), "three_d": (16, 16, 16, 1)},
                {"one_d": (16, 1), "two_d": (16, 16, 1), "three_d": (16, 16, 16, 1)}):   # exactly one of the three shapes
        try:
            dfft.LinesConvolvePlan(**bad)
            raise AssertionError(bad)
        except ValueError:
            pass
    n, nlines = 256, 6
    for real in (False, True):
        for prec in (dfft.DOUBLE, dfft.FLOAT):
            rsz = 4 if prec == dfft.FLOAT else 8
            csz = 2 * rsz
            esz = rsz if real else csz
            io = n * nlines * esz
            mb = (n // 2 + 1 if real else n) * csz
            a, b, m = alloc(io + 64), alloc(io + 64), alloc(mb * nlines + 64)
            p = dfft.LinesConvolvePlan(one_d=(n, nlines), precision=prec, real=real)
            assert code(lambda: p.execute(a, b, m, 1)) == 0
            assert code(lambda: p.execute(a, a, m, nlines)) == 0                            # in place
            assert code(lambda: p.execute(a + 16 * esz, a, m)) == -1                        # partial overlap of in and out
            assert code(lambda: p.execute(a, a + 16 * esz, m)) == -1
            assert code(lambda: p.execute(a, b, b)) == -1                                   # multiplier overlaps out
            assert code(lambda: p.execute(a, b, b + io - csz)) == -1
            assert code(lambda: p.execute(a, b, b + io)) == 0                               # right after out
            assert code(lambda: p.execute(a, b, a)) == 0                                    # the multiplier may share `in`
            assert code(lambda: p.execute(None, b, m)) == -1
            assert code(lambda: p.execute(a, None, m)) == -1
            assert code(lambda: p.execute(a, b, None)) == -1
            for mc in (0, 2, nlines + 1, -1):
                assert code(lambda: p.execute(a, b, m, mc)) == -1, mc
            assert code(lambda: p.execute(a + esz // 2, b, m)) == -1                        # misaligned in / out / multiplier
            assert code(lambda: p.execute(a, b + esz // 2, m)) == -1
            assert code(lambda: p.execute(a, b, m + rsz)) == -1
            if prec == dfft.FLOAT and not real:
                assert code(lambda: p.execute(a + 8, b + 8, m + 8)) == 0                    # fp32 complex at an odd complex64 offset
            # the other execute entry points refuse a convolve plan
            assert code(lambda: dfft.api._check(L.dfft_lines_execute(p.handle, a, dfft.FORWARD), "x")) == -1
            assert code(lambda: dfft.api._check(L.dfft_lines_execute_real(p.handle, a, b, dfft.FORWARD), "x")) == -1
            p.synchronize(); p.destroy()
            for q in (a, b, m):
                L.dfft_free_local(q, dfft.ALLOC_DEV)
    # and dfft_lines_execute_convolve refuses the 1-D lines plans
    d = alloc(n * nlines * 16 * 2)
    for other in (dfft.LinesPlan(n, 1, nlines, nlines, n, 0), dfft.RealLinesPlan(n, nlines)):
        assert code(lambda: dfft.api._check(L.dfft_lines_execute_convolve(other.handle, d, d, d + n * nlines * 16, 1), "x")) == -1
        other.destroy()
    L.dfft_free_local(d, dfft.ALLOC_DEV)
    assert L.fakecuda_live_allocations() == 0, ("leak", L.fakecuda_live_allocations())
    print("1-D convolve lines fakecuda control flow ok")
''')


def test_1d_convolve_lines_plans_run_to_completion_on_a_fake_runtime(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, DFFT_VERBOSE="1")
    for var in ("DFFT_NO_PLANE", "DFFT_FORCE_PLANE", "DFFT_GENERIC", "DFFT_VARIANT"):
        env.pop(var, None)
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "1-D convolve lines fakecuda control flow ok" in r.stdout
