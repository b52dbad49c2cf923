"""CPU test of the non-dry host control flow of the batched 2-D convolve lines plans (dfft_lines_plan_create_convolve_2d /
_r2c_2d), on the fake CUDA runtime of test_control_flow_fakecuda.py (device memory = host memory, launches = counted no-ops):
create -> 3 executes -> destroy in both precisions, with 1 launch per execute where the one-kernel convolution of square
images runs and 3 otherwise (DFFT_NO_PLANE=1, other shapes, R2C), nothing left allocated, and every execute-time rejection
coming back as its error code."""
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
        nx, ny, batch = shape
        rsz = 4 if precision == dfft.FLOAT else 8
        img = nx * ny
        io = img * batch * (rsz if real else 2 * rsz)
        mimg = ny * (nx // 2 + 1 if real else nx)
        a, b, m = alloc(io), alloc(io), alloc(mimg * batch * 2 * rsz)
        plan = dfft.LinesConvolvePlan(two_d=shape, precision=precision, real=real, flags=flags)
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
            # the table may leave an instantiation off; the launches follow the recorded passes, and DFFT_FORCE_PLANE=1 runs it
            default = len(dfft.lines_conv_2d_ops(n, n, 5, prec))
            assert default in (1, 3), default
            drive(prec, (n, n, 5), False, default)
            drive(prec, (n, n, 2), False, default, dfft.SCALE_BACKWARD)
            os.environ["DFFT_FORCE_PLANE"] = "1"
            drive(prec, (n, n, 5), False, 1)
            drive(prec, (n, n, 3), False, 1, dfft.SCALE_BACKWARD)
            del os.environ["DFFT_FORCE_PLANE"]
            os.environ["DFFT_NO_PLANE"] = "1"
            drive(prec, (n, n, 5), False, 3)
            del os.environ["DFFT_NO_PLANE"]
            drive(prec, (n, n, 5), True, 3)
        for shape in ((48, 48, 2), (16, 8, 3), (14, 16, 1), (9, 9, 2), (12, 125, 1), (64, 32, 2)):
            drive(prec, shape, False, 3)
            drive(prec, shape, True, 3)

    def code(fn):
        try:
            fn()
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0])
        return 0

    assert code(lambda: dfft.LinesConvolvePlan(two_d=(16, 14, 1)).destroy()) == -3            # no tuned y kernel
    assert code(lambda: dfft.LinesConvolvePlan(two_d=(16, 16, 1), flags=dfft.NO_FUSE).destroy()) == -1
    assert code(lambda: dfft.LinesConvolvePlan(two_d=(16, 16, 1 << 27), real=True).destroy()) == -3
    assert code(lambda: dfft.LinesConvolvePlan(two_d=(16, 16, 1 << 27)).destroy()) == -3
    assert code(lambda: dfft.api._check(L.dfft_lines_plan_create_convolve_2d(16, 16, 1, dfft.DOUBLE, 0, None), "x")) == -1
    assert code(lambda: dfft.api._check(L.dfft_lines_plan_create_convolve_r2c_2d(16, 16, 1, dfft.DOUBLE, 0, None), "x")) == -1
    for bad in ({}, {"two_d": (16, 16, 1), "three_d": (16, 16, 16, 1)}):                       # exactly one of the two shapes
        try:
            dfft.LinesConvolvePlan(**bad)
            raise AssertionError(bad)
        except ValueError:
            pass
    nx, ny, batch = 16, 16, 5
    img = nx * ny
    for env in ("DFFT_FORCE_PLANE", "DFFT_NO_PLANE"):
        os.environ[env] = "1"
        for real in (False, True):
            for prec in (dfft.DOUBLE, dfft.FLOAT):
                rsz = 4 if prec == dfft.FLOAT else 8
                csz = 2 * rsz
                esz = rsz if real else csz
                io = img * batch * esz
                mb = ny * (nx // 2 + 1 if real else nx) * csz
                a, b, m = alloc(io + 64), alloc(io + 64), alloc(mb * batch + 64)
                p = dfft.LinesConvolvePlan(two_d=(nx, ny, batch), precision=prec, real=real)
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
        del os.environ[env]
    # and dfft_lines_execute_convolve refuses the 2-D lines plans
    d = alloc(img * batch * 16 * 2)
    for other in (dfft.LinesPlan(two_d=(nx, ny, batch)), dfft.RealLinesPlan(two_d=(nx, ny, batch))):
        assert code(lambda: dfft.api._check(L.dfft_lines_execute_convolve(other.handle, d, d, d + img * batch * 16, 1), "x")) == -1
        other.destroy()
    L.dfft_free_local(d, dfft.ALLOC_DEV)
    assert L.fakecuda_live_allocations() == 0, ("leak", L.fakecuda_live_allocations())
    print("2-D convolve lines fakecuda control flow ok")
''')


def test_2d_convolve_lines_plans_run_to_completion_on_a_fake_runtime(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, DFFT_VERBOSE="1")
    for var in ("DFFT_NO_PLANE", "DFFT_FORCE_PLANE", "DFFT_GENERIC", "DFFT_VARIANT"):
        env.pop(var, None)
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "2-D convolve lines fakecuda control flow ok" in r.stdout
