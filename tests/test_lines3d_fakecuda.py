"""CPU test of the non-dry host control flow of the batched 3-D lines plans (dfft_lines_plan_create_3d / _r2c_3d), on the fake
CUDA runtime of test_control_flow_fakecuda.py (device memory = host memory, launches = counted no-ops): create -> 3 executes per
direction -> destroy in both precisions, with 2 launches per execute where the plane kernel runs (X + Y in one), 3 without it
and 3 for real plans, nothing left allocated, and every execute-time rejection coming back as its error code."""
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

    def count(plan, runs):
        l0, e0 = L.fakecuda_launches(), L.fakecuda_event_records()
        for args in runs:
            for _ in range(3):
                plan.execute(*args)
        plan.synchronize()
        assert L.fakecuda_event_records() - e0 >= 6 * len(runs)   # start and end event of every execute
        return (L.fakecuda_launches() - l0) // (3 * len(runs))

    def drive_c2c(precision, shape, want):
        nx, ny, nz, batch = shape
        esz = 8 if precision == dfft.FLOAT else 16
        d = alloc(nx * ny * nz * batch * esz)
        plan = dfft.LinesPlan(three_d=shape, precision=precision)
        got = count(plan, [(d, dfft.FORWARD), (d, dfft.BACKWARD)])
        assert got == want, (shape, precision, got, want)
        assert plan.stream
        plan.destroy()
        L.dfft_free_local(d, dfft.ALLOC_DEV)

    def drive_real(precision, shape):
        nx, ny, nz, batch = shape
        rsz = 4 if precision == dfft.FLOAT else 8
        rows = ny * nz * batch
        r, c = alloc(rows * nx * rsz), alloc(rows * (nx // 2 + 1) * 2 * rsz)
        plan = dfft.RealLinesPlan(three_d=shape, precision=precision)
        assert count(plan, [(r, c, dfft.FORWARD)]) == 3 and count(plan, [(c, r, dfft.BACKWARD)]) == 3, shape
        plan.destroy()
        L.dfft_free_local(r, dfft.ALLOC_DEV); L.dfft_free_local(c, dfft.ALLOC_DEV)

    for prec in (dfft.DOUBLE, dfft.FLOAT):
        for n in (16, 32, 64):
            drive_c2c(prec, (n, n, 8, 3), 2)
            os.environ["DFFT_NO_PLANE"] = "1"
            drive_c2c(prec, (n, n, 8, 3), 3)
            del os.environ["DFFT_NO_PLANE"]
        for shape in ((48, 48, 4, 2), (16, 8, 4, 3), (14, 22, 26, 1), (9, 9, 9, 2)):
            drive_c2c(prec, shape, 3)
        for shape in ((64, 64, 64, 1), (16, 16, 16, 3), (9, 8, 6, 3), (14, 12, 10, 2), (360, 6, 4, 1)):
            drive_real(prec, shape)

    def code(fn):
        try:
            fn()
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0])
        return 0

    assert code(lambda: dfft.LinesPlan(three_d=(17, 16, 16, 1)).destroy()) == -3
    assert code(lambda: dfft.LinesPlan(three_d=(16, 16, 16, 1 << 23)).destroy()) == -3
    assert code(lambda: dfft.RealLinesPlan(three_d=(16, 16, 16, 1 << 23)).destroy()) == -3
    assert code(lambda: dfft.LinesPlan(three_d=(16, 16, 0, 1)).destroy()) == -1
    assert code(lambda: dfft.api._check(L.dfft_lines_plan_create_3d(16, 16, 16, 1, dfft.DOUBLE, None), "x")) == -1
    # complex plan: null data, bad direction, the real execute
    nx, ny, nz, batch = 16, 16, 4, 2
    d = alloc(nx * ny * nz * batch * 16 + 64)
    p = dfft.LinesPlan(three_d=(nx, ny, nz, batch))
    assert code(lambda: p.execute(d, dfft.FORWARD)) == 0
    assert code(lambda: p.execute(None, dfft.FORWARD)) == -1
    assert code(lambda: p.execute(d, 0)) == -1
    assert code(lambda: dfft.api._check(L.dfft_lines_execute_real(p.handle, d, d + 8192, dfft.FORWARD), "x")) == -1
    q = dfft.LinesPlan(three_d=(nx, ny, nz, batch), precision=dfft.FLOAT)
    assert code(lambda: q.execute(d + 8, dfft.FORWARD)) == 0       # fp32 complex at an odd complex64 offset
    p.synchronize(); p.destroy(); q.synchronize(); q.destroy()
    # real plan: overlap, alignment, null pointers, the complex execute
    H = nx // 2 + 1
    rows = ny * nz * batch
    r, c = alloc(rows * nx * 8 + 64), alloc(rows * H * 16 + 64)
    p = dfft.RealLinesPlan(three_d=(nx, ny, nz, batch))
    assert code(lambda: p.execute(r, c, dfft.FORWARD)) == 0
    assert code(lambda: p.execute(c, r, dfft.BACKWARD)) == 0
    assert code(lambda: p.execute(r, r, dfft.FORWARD)) == -1                       # in == out
    assert code(lambda: p.execute(r, r + 8 * 16, dfft.FORWARD)) == -1              # overlapping ranges
    assert code(lambda: p.execute(r, c + 8, dfft.FORWARD)) == -1                   # fp64 complex output not 16-byte aligned
    assert code(lambda: p.execute(c + 8, r, dfft.BACKWARD)) == -1
    assert code(lambda: p.execute(r + 4, c, dfft.FORWARD)) == -1                   # real fp64 not 8-byte aligned
    assert code(lambda: p.execute(None, c, dfft.FORWARD)) == -1
    assert code(lambda: p.execute(r, None, dfft.FORWARD)) == -1
    assert code(lambda: p.execute(r, c, 0)) == -1
    assert code(lambda: dfft.api._check(L.dfft_lines_execute(p.handle, r, dfft.FORWARD), "x")) == -1   # real plan, C2C execute
    p.synchronize(); p.destroy()
    L.dfft_free_local(d, dfft.ALLOC_DEV); L.dfft_free_local(r, dfft.ALLOC_DEV); L.dfft_free_local(c, dfft.ALLOC_DEV)
    assert L.fakecuda_live_allocations() == 0, ("leak", L.fakecuda_live_allocations())
    print("3-D lines fakecuda control flow ok")
''')


def test_3d_lines_plans_run_to_completion_on_a_fake_runtime(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, DFFT_VERBOSE="1")
    env.pop("DFFT_NO_PLANE", None)
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "3-D lines fakecuda control flow ok" in r.stdout
