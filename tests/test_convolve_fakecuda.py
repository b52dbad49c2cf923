"""CPU test of the non-dry host control flow of the spectral convolution plans (dfft_plan_convolve_*).

The library's objects are linked against tests/fakecuda/fake_cudart.cpp as in test_control_flow_fakecuda.py (device memory =
host memory, launches = counted no-ops).  Plans of 1, 2 and 4 device-threads run create -> three executes with different
multipliers -> timings -> destroy, C2C and R2C, P2P and NCCL-free modes, with nothing left allocated afterwards; every
execute-time rejection comes back as its error code; and with FAKECUDA_TMA=1 (a cuTensorMapEncodeTiled stand-in that enforces the
driver's constraints) under DFFT_TMA=2 every map a convolve plan encodes is accepted."""
import os
import subprocess
import sys
import textwrap

from test_control_flow_fakecuda import ROOT, fake_lib  # noqa: F401  (fixture)

WORKER = textwrap.dedent(r'''
    import ctypes, os, sys, threading
    sys.path.insert(0, sys.argv[1])
    import distributedfft_b200.api as api
    api.LIB_PATH = sys.argv[2]
    api._lib = None
    import distributedfft_b200 as dfft
    L = dfft.lib()
    L.fakecuda_launches.restype = ctypes.c_longlong
    L.fakecuda_live_allocations.restype = ctypes.c_longlong
    L.fakecuda_tma_maps.restype = ctypes.c_longlong
    L.fakecuda_tma_maps.argtypes = [ctypes.c_void_p, ctypes.c_longlong]

    def drive(n0, n1, n2, P, flags, precision=dfft.DOUBLE, real=False, executes=3, inplace=False):
        comm = dfft.LocalComm(P) if P > 1 else None
        errs = []
        def worker(p):
            try:
                _, ln0, _, ln1, _ = dfft.fft_mpi_local_size_3d(n0, n1, n2, P, p)
                cnt = ln0 * n1 * n2
                words = (cnt + 1) // 2 if real else cnt          # allocation unit: one complex element
                a = dfft.fft_mpi_alloc_local_memory(words, dfft.ALLOC_DEV, precision)
                b = None if inplace else dfft.fft_mpi_alloc_local_memory(words, dfft.ALLOC_DEV, precision)
                mults = [dfft.fft_mpi_alloc_local_memory(n0 * ln1 * (n2 // 2 + 1 if real else n2), dfft.ALLOC_DEV, precision) for _ in range(3)]
                plan = dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, a, b, comm, p, P, precision, flags, real=real)
                assert (plan.in_count, plan.out_count) == (cnt, cnt)
                assert plan.pipeline_parts == 0
                for k in range(executes):
                    plan.execute_convolve(mults[k % 3])
                plan.synchronize()
                t = plan.timings(); pt = plan.pass_timings()
                assert len(t) == 5 and len(pt) == 3 and t[1] == 0 and plan.launches >= 3
                plan.destroy()
                for x in [a, b] + mults:
                    if x: L.dfft_free_local(x, dfft.ALLOC_DEV)
            except Exception:
                import traceback
                errs.append(traceback.format_exc())
        if P == 1:
            worker(0)
        else:
            th = [threading.Thread(target=worker, args=(p,)) for p in range(P)]
            [t.start() for t in th]; [t.join() for t in th]
        if comm: comm.destroy()
        assert not errs, "\n".join(errs)

    before = L.fakecuda_launches()
    for real in (False, True):
        for flags in (0, dfft.SCALE_BACKWARD, dfft.NO_FUSE | dfft.NO_TMA, dfft.FORCE_FUSE, dfft.FORCE_PIPELINE | dfft.OVERLAP_X):
            drive(64, 64, 64, 1, flags, real=real)
            drive(8, 6, 9, 1, flags, dfft.FLOAT, real=real, inplace=True)
        for P in (2, 4):
            for flags in (dfft.EXCHANGE_P2P, dfft.EXCHANGE_P2P | dfft.SCALE_BACKWARD, dfft.EXCHANGE_P2P | dfft.NO_FUSE):
                drive(64, 64, 64, P, flags, real=real)
                drive(10, 12, 9, P, flags, real=real)       # uneven split, odd z length
    # execute-time rejections on the real path
    def code(fn):
        try:
            fn()
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0])
        return 0
    d = dfft.fft_mpi_alloc_local_memory(16 * 16 * 16, dfft.ALLOC_DEV)
    h = dfft.fft_mpi_alloc_local_memory(16 * 16 * 16, dfft.ALLOC_CPU)
    m = dfft.fft_mpi_alloc_local_memory(16 * 16 * 16, dfft.ALLOC_DEV)
    p = dfft.fft_mpi_plan_dft_convolve_3d(16, 16, 16, d, None, None, 0, 1)
    assert code(p.execute) == -1
    assert code(lambda: p.execute_stage(0)) == -1
    assert code(lambda: p.execute_host(h, h)) == -1
    assert code(lambda: p.execute_host_async(h, h)) == -1
    assert code(lambda: p.execute_convolve(None)) == -1
    assert code(lambda: p.execute_convolve(m + 8)) == -1
    assert code(lambda: p.execute_convolve(m)) == 0
    p.synchronize(); p.destroy()
    q = dfft.fft_mpi_plan_dft_c2c_3d(16, 16, 16, d, None, None, 0, 1, dfft.FORWARD)
    assert code(lambda: q.execute_convolve(m)) == -1
    q.destroy()
    L.dfft_free_local(d, dfft.ALLOC_DEV); L.dfft_free_local(m, dfft.ALLOC_DEV); L.dfft_free_local(h, dfft.ALLOC_CPU)
    # TMA: every map a convolve plan encodes passes the driver's constraints (DFFT_TMA=2 turns every pass mode on)
    os.environ["DFFT_TMA"] = "2"
    L.fakecuda_tma_reset()
    for shape in ((8, 512, 512), (8, 256, 256), (4, 1024, 243), (16, 768, 125), (256, 256, 16)):
        for prec in (dfft.DOUBLE, dfft.FLOAT):
            for real in (False, True):
                drive(*shape, 1, 0, prec, real=real, executes=1)
    drive(16, 512, 512, 2, dfft.EXCHANGE_P2P, executes=1)
    print("tma maps encoded: %d" % L.fakecuda_tma_maps(None, 0))
    assert L.fakecuda_tma_maps(None, 0) > 0
    assert L.fakecuda_launches() - before > 50
    assert L.fakecuda_live_allocations() == 0, ("leak", L.fakecuda_live_allocations())
    print("convolve fakecuda control flow ok")
''')


def test_convolve_plans_run_to_completion_on_a_fake_runtime(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, DFFT_VERBOSE="1", FAKECUDA_TMA="1")
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "convolve fakecuda control flow ok" in r.stdout
