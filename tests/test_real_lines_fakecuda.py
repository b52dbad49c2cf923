"""CPU test of the non-dry host control flow of the real lines plans (dfft_lines_plan_create_r2c / _r2c_2d,
dfft_lines_execute_real), on the fake CUDA runtime of test_control_flow_fakecuda.py (device memory = host memory, launches =
counted no-ops): create -> 3 executes per direction -> destroy for 1-D and 2-D plans, tuned and run-time-scheduled lengths,
both precisions, with one launch per execute for 1-D and two for 2-D and nothing left allocated; and every rejection comes back
as its error code on the real path."""
import os
import subprocess
import sys
import textwrap

from test_control_flow_fakecuda import ROOT, fake_lib  # noqa: F401  (fixture)

WORKER = textwrap.dedent(r'''
    import ctypes, sys
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

    def drive(precision, n=None, nlines=0, two_d=None):
        rsz = 4 if precision == dfft.FLOAT else 8
        rows = nlines if two_d is None else two_d[1] * two_d[2]
        nx = n if two_d is None else two_d[0]
        r, c = alloc(rows * nx * rsz), alloc(rows * (nx // 2 + 1) * 2 * rsz)
        plan = dfft.RealLinesPlan(n, nlines, precision, two_d)
        per = 1 if two_d is None else 2
        for direction, i, o in ((dfft.FORWARD, r, c), (dfft.BACKWARD, c, r)):
            l0, e0 = L.fakecuda_launches(), L.fakecuda_event_records()
            for _ in range(3):
                plan.execute(i, o, direction)
            plan.synchronize()
            assert L.fakecuda_launches() - l0 == 3 * per, (n, two_d, direction, L.fakecuda_launches() - l0)
            assert L.fakecuda_event_records() - e0 >= 6          # start and end event of every execute
        assert plan.stream
        plan.destroy()
        L.dfft_free_local(r, dfft.ALLOC_DEV); L.dfft_free_local(c, dfft.ALLOC_DEV)

    for prec in (dfft.DOUBLE, dfft.FLOAT):
        for n, nlines in ((512, 9), (64, 100), (9, 7), (14, 5), (360, 1), (2, 3), (13, 8)):
            drive(prec, n, nlines)
        for nx, ny, batch in ((1024, 64, 2), (9, 8, 3), (14, 12, 2), (16, 14, 1), (480, 22, 3)):
            drive(prec, two_d=(nx, ny, batch))
    assert dfft.length_kind(360) == 1 and dfft.length_kind(14) == 1 and dfft.length_kind(512) == 2

    def code(fn):
        try:
            fn()
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0])
        return 0

    # lengths and line counts
    for n in (17, 1, 8192):
        assert code(lambda: dfft.RealLinesPlan(n, 4).destroy()) == -3, n
    assert code(lambda: dfft.RealLinesPlan(16, 1 << 31).destroy()) == -3
    assert code(lambda: dfft.RealLinesPlan(two_d=(16, 1 << 16, 1 << 15)).destroy()) == -3
    assert code(lambda: dfft.RealLinesPlan(two_d=(16, 17, 2)).destroy()) == -3
    # buffers
    n, nlines = 16, 6
    r, c = alloc(nlines * n * 8 + 64), alloc(nlines * (n // 2 + 1) * 16 + 64)
    p = dfft.RealLinesPlan(n, nlines)
    assert code(lambda: p.execute(r, c, dfft.FORWARD)) == 0
    assert code(lambda: p.execute(c, r, dfft.BACKWARD)) == 0
    assert code(lambda: p.execute(r, r, dfft.FORWARD)) == -1                       # in == out
    assert code(lambda: p.execute(r, r + 8 * 16, dfft.FORWARD)) == -1              # overlapping ranges
    assert code(lambda: p.execute(r + 8 * 16, r, dfft.BACKWARD)) == -1
    assert code(lambda: p.execute(r, c + 8, dfft.FORWARD)) == -1                   # fp64 complex output not 16-byte aligned
    assert code(lambda: p.execute(c + 8, r, dfft.BACKWARD)) == -1                  # ... complex input
    assert code(lambda: p.execute(r + 8, c, dfft.FORWARD)) == 0                    # a real fp64 buffer needs 8 bytes
    assert code(lambda: p.execute(r + 4, c, dfft.FORWARD)) == -1
    assert code(lambda: p.execute(None, c, dfft.FORWARD)) == -1                    # null pointers
    assert code(lambda: p.execute(r, None, dfft.FORWARD)) == -1
    assert code(lambda: p.execute(r, c, 0)) == -1                                  # bad direction
    assert code(lambda: dfft.api._check(L.dfft_lines_execute(p.handle, r, dfft.FORWARD), "x")) == -1   # real plan, C2C execute
    p.synchronize(); p.destroy()
    q = dfft.RealLinesPlan(9, 5, dfft.FLOAT)
    assert code(lambda: q.execute(r, c + 8, dfft.FORWARD)) == 0                    # fp32 complex at an odd complex64 offset
    q.destroy()
    cp = dfft.LinesPlan(16, 1, 4, 4, 16, 0)
    assert code(lambda: dfft.api._check(L.dfft_lines_execute_real(cp.handle, r, c, dfft.FORWARD), "x")) == -1
    cp.destroy()
    L.dfft_free_local(r, dfft.ALLOC_DEV); L.dfft_free_local(c, dfft.ALLOC_DEV)
    assert L.fakecuda_live_allocations() == 0, ("leak", L.fakecuda_live_allocations())
    print("real lines fakecuda control flow ok")
''')


def test_real_lines_plans_run_to_completion_on_a_fake_runtime(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, DFFT_VERBOSE="1")
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "real lines fakecuda control flow ok" in r.stdout
