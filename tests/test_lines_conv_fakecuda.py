"""CPU test of the non-dry host control flow of the batched 3-D convolve lines plans (dfft_lines_plan_create_convolve_3d /
_r2c_3d), on the fake CUDA runtime of test_control_flow_fakecuda.py (device memory = host memory, launches = counted no-ops):
create -> 3 executes -> destroy in both precisions, with 3 launches per execute where the plane kernel runs and 5 otherwise
(also under DFFT_NO_PLANE=1), nothing left allocated, and every execute-time rejection coming back as its error code."""
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

    def drive(precision, shape, real, want, flags=0):
        nx, ny, nz, batch = shape
        rsz = 4 if precision == dfft.FLOAT else 8
        vol = nx * ny * nz
        io = vol * batch * (rsz if real else 2 * rsz)
        mvol = nz * ny * (nx // 2 + 1 if real else nx)
        a, b, m = alloc(io), alloc(io), alloc(mvol * batch * 2 * rsz)
        plan = dfft.LinesConvolvePlan(shape, precision=precision, real=real, flags=flags)
        l0, e0 = L.fakecuda_launches(), L.fakecuda_event_records()
        plan.execute(a, b, m, 1)
        plan.execute(a, a, m, batch)
        plan.execute(b, a, m, 1)
        plan.synchronize()
        assert L.fakecuda_event_records() - e0 >= 6              # start and end event of every execute
        got = (L.fakecuda_launches() - l0) // 3
        assert got == want, (shape, precision, real, got, want)
        assert plan.stream
        plan.destroy()
        for p in (a, b, m):
            L.dfft_free_local(p, dfft.ALLOC_DEV)

    for prec in (dfft.DOUBLE, dfft.FLOAT):
        for n in (16, 32, 64):
            drive(prec, (n, n, 16, 3), False, 3)
            drive(prec, (n, n, 32, 2), False, 3, dfft.SCALE_BACKWARD)
            os.environ["DFFT_NO_PLANE"] = "1"
            drive(prec, (n, n, 16, 3), False, 5)
            del os.environ["DFFT_NO_PLANE"]
            drive(prec, (n, n, 16, 3), True, 5)
        for shape in ((48, 48, 12, 2), (16, 8, 32, 3), (14, 22, 16, 1), (9, 9, 9, 2), (12, 10, 125, 1)):
            drive(prec, shape, False, 5)
            drive(prec, shape, True, 5)

    def code(fn):
        try:
            fn()
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0])
        return 0

    assert code(lambda: dfft.LinesConvolvePlan((16, 16, 14, 1)).destroy()) == -3            # no tuned z kernel
    assert code(lambda: dfft.LinesConvolvePlan((16, 16, 16, 1), flags=dfft.NO_FUSE).destroy()) == -1
    assert code(lambda: dfft.LinesConvolvePlan((16, 16, 16, 1 << 23), real=True).destroy()) == -3
    assert code(lambda: dfft.api._check(L.dfft_lines_plan_create_convolve_3d(16, 16, 16, 1, dfft.DOUBLE, 0, None), "x")) == -1
    nx, ny, nz, batch = 16, 16, 8, 4
    vol = nx * ny * nz
    for real in (False, True):
        for prec in (dfft.DOUBLE, dfft.FLOAT):
            rsz = 4 if prec == dfft.FLOAT else 8
            csz = 2 * rsz
            esz = rsz if real else csz
            io = vol * batch * esz
            mb = nz * ny * (nx // 2 + 1 if real else nx) * csz
            a, b, m = alloc(io + 64), alloc(io + 64), alloc(mb * batch + 64)
            p = dfft.LinesConvolvePlan((nx, ny, nz, batch), precision=prec, real=real)
            assert code(lambda: p.execute(a, b, m, 1)) == 0
            assert code(lambda: p.execute(a, a, m, batch)) == 0                             # in place
            assert code(lambda: p.execute(a + 16 * esz, a, m)) == -1                        # partial overlap of in and out
            assert code(lambda: p.execute(a, a + 16 * esz, m)) == -1
            assert code(lambda: p.execute(a, b, b)) == -1                                   # multiplier overlaps out
            assert code(lambda: p.execute(a, b, b + io - csz)) == -1
            assert code(lambda: p.execute(a, b, b + io)) == 0                               # right after out
            assert code(lambda: p.execute(a, b, a)) == 0                                    # the multiplier may share `in`
            assert code(lambda: p.execute(None, b, m)) == -1
            assert code(lambda: p.execute(a, None, m)) == -1
            assert code(lambda: p.execute(a, b, None)) == -1
            for mc in (0, 2, batch + 1, -1):
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
    # and dfft_lines_execute_convolve refuses every other lines plan
    d = alloc(vol * batch * 16 * 2)
    for other in (dfft.LinesPlan(three_d=(nx, ny, nz, batch)), dfft.RealLinesPlan(three_d=(nx, ny, nz, batch)), dfft.LinesPlan(two_d=(nx, ny, batch))):
        assert code(lambda: dfft.api._check(L.dfft_lines_execute_convolve(other.handle, d, d, d + vol * batch * 16, 1), "x")) == -1
        other.destroy()
    L.dfft_free_local(d, dfft.ALLOC_DEV)
    assert L.fakecuda_live_allocations() == 0, ("leak", L.fakecuda_live_allocations())
    print("3-D convolve lines fakecuda control flow ok")
''')


def test_3d_convolve_lines_plans_run_to_completion_on_a_fake_runtime(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, DFFT_VERBOSE="1")
    for var in ("DFFT_NO_PLANE", "DFFT_FORCE_PLANE", "DFFT_GENERIC", "DFFT_VARIANT"):
        env.pop(var, None)
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "3-D convolve lines fakecuda control flow ok" in r.stdout
