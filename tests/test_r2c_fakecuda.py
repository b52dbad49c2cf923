"""CPU test of the non-dry host control flow of R2C / C2R plans (dfft_plan_r2c_3d).

The library's objects are linked against tests/fakecuda/fake_cudart.cpp as in test_control_flow_fakecuda.py (device memory =
host memory, launches = counted no-ops).  Real plans of 1, 2 and 4 device-threads run create -> 3 executes -> timings ->
destroy in both directions, P2P and NCCL-free modes, with nothing left allocated afterwards; every unsupported request comes
back as its error code on the real path too; and with FAKECUDA_TMA=1 (a cuTensorMapEncodeTiled stand-in that enforces the
driver's constraints) under DFFT_TMA=2 every map an R2C plan encodes is accepted."""
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

    def drive(n0, n1, n2, P, flags, precision=dfft.DOUBLE, executes=3):
        comm = dfft.LocalComm(P) if P > 1 else None
        errs, masks = [], []
        def worker(p):
            try:
                rc, cc = dfft.local_size_r2c_3d(n0, n1, n2, P, p)
                for direction in (dfft.FORWARD, dfft.BACKWARD):
                    ni, no = (rc, cc) if direction == dfft.FORWARD else (cc, rc)
                    ri = direction == dfft.FORWARD
                    a = dfft.fft_mpi_alloc_local_memory((ni + 1) // 2 if ri else ni, dfft.ALLOC_DEV, precision)
                    b = dfft.fft_mpi_alloc_local_memory(no if ri else (no + 1) // 2, dfft.ALLOC_DEV, precision)
                    plan = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, a, b, comm, p, P, direction, precision, flags)
                    assert (plan.in_count, plan.out_count) == (ni, no)
                    assert not plan.fused and plan.pipeline_parts == 0
                    for _ in range(executes):
                        plan.execute()
                    plan.synchronize()
                    t = plan.timings(); pt = plan.pass_timings()
                    assert len(t) == 5 and len(pt) == 3 and plan.launches >= 3
                    masks.append(plan.tma_mask)
                    plan.destroy()
                    L.dfft_free_local(a, dfft.ALLOC_DEV); L.dfft_free_local(b, dfft.ALLOC_DEV)
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
        return masks

    before = L.fakecuda_launches()
    for flags in (0, dfft.SCALE_BACKWARD, dfft.NATURAL_SPECTRUM, dfft.FORCE_FUSE | dfft.OVERLAP_X | dfft.FORCE_PIPELINE, dfft.NO_TMA):
        drive(64, 64, 64, 1, flags)
        drive(5, 7, 9, 1, flags, dfft.FLOAT)
    for P in (2, 4):
        for flags in (dfft.EXCHANGE_P2P, dfft.EXCHANGE_P2P | dfft.SCALE_BACKWARD, dfft.EXCHANGE_P2P | dfft.FORCE_PIPELINE):
            drive(64, 64, 64, P, flags)
            drive(10, 10, 243, P, flags)         # uneven split, odd z length
    # host entry points: real and complex slab sizes
    rc, cc = dfft.local_size_r2c_3d(16, 12, 10, 1, 0)
    d_r = dfft.fft_mpi_alloc_local_memory((rc + 1) // 2, dfft.ALLOC_DEV); d_c = dfft.fft_mpi_alloc_local_memory(cc, dfft.ALLOC_DEV)
    h_r = dfft.fft_mpi_alloc_local_memory((rc + 1) // 2, dfft.ALLOC_CPU); h_c = dfft.fft_mpi_alloc_local_memory(cc, dfft.ALLOC_CPU)
    for direction, i, o, hi, ho in ((dfft.FORWARD, d_r, d_c, h_r, h_c), (dfft.BACKWARD, d_c, d_r, h_c, h_r)):
        plan = dfft.fft_mpi_plan_dft_r2c_3d(16, 12, 10, i, o, None, 0, 1, direction)
        plan.execute_host(hi, ho); plan.execute_host_async(hi, ho); plan.synchronize(); plan.destroy()
    # rejections on the real path
    def code(fn):
        try:
            fn()
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0])
        return 0
    def mk(n2=16, inp=d_c, out=d_r, flags=0, prec=dfft.DOUBLE, direction=dfft.FORWARD):
        return lambda: dfft.fft_mpi_plan_dft_r2c_3d(8, 8, n2, inp, out, None, 0, 1, direction, prec, flags).destroy()
    assert code(mk(out=None)) == -1 and code(mk(out=d_c)) == -1                # in place
    assert code(mk(flags=dfft.EXCHANGE_STAGED)) == -3                          # staged
    assert code(mk(n2=14)) == -3                                               # generic z length
    assert code(mk(inp=d_r, out=d_c + 8)) == -1                                # misaligned fp64 complex output
    p = dfft.fft_mpi_plan_dft_r2c_3d(8, 8, 16, d_r, d_c, None, 0, 1, dfft.FORWARD)
    assert code(lambda: p.execute_stage(0)) == -3
    p.destroy()
    for x in (d_r, d_c): L.dfft_free_local(x, dfft.ALLOC_DEV)
    for x in (h_r, h_c): L.dfft_free_local(x, dfft.ALLOC_CPU)
    # TMA: every map an R2C plan encodes passes the driver's constraints (DFFT_TMA=2 turns every pass mode on)
    os.environ["DFFT_TMA"] = "2"
    L.fakecuda_tma_reset()
    for shape in ((8, 512, 512), (8, 256, 256), (4, 1024, 243), (16, 768, 125)):
        for prec in (dfft.DOUBLE, dfft.FLOAT):
            drive(*shape, 1, 0, prec, executes=1)
    drive(16, 512, 512, 2, dfft.EXCHANGE_P2P, executes=1)
    print("tma maps encoded: %d" % L.fakecuda_tma_maps(None, 0))
    assert L.fakecuda_launches() - before > 50
    assert L.fakecuda_live_allocations() == 0, ("leak", L.fakecuda_live_allocations())
    print("r2c fakecuda control flow ok")
''')


def test_r2c_plans_run_to_completion_on_a_fake_runtime(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, DFFT_VERBOSE="1", FAKECUDA_TMA="1")
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "r2c fakecuda control flow ok" in r.stdout
