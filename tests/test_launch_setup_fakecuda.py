"""CPU test of the launch set-up every pass-kernel launcher shares (dfft_launch.cuh), on the fake CUDA runtime of
test_control_flow_fakecuda.py, which records per (device, kernel) the dynamic shared-memory opt-ins, the occupancy queries and the
launches, and refuses a launch above 48 KiB of dynamic shared memory that the device's opt-in for the kernel does not cover.

Two device-threads of one LocalComm sit on fake devices 0 and 1 and run TMA kernels (16 x 512 x 512 fp32 over P2P, forward,
two-sweep t0); then a 3-D lines plan (plane kernel) and a 2-D convolve lines plan run twice each.  Every execute must succeed,
each pass kernel must have had its opt-in exactly once on each device it ran on, and each tuned kernel at most one occupancy
query there (the run-time-scheduled fft_generic_* kernels query theirs at every launch)."""
import os
import re
import subprocess
import sys
import textwrap

from test_control_flow_fakecuda import ROOT, fake_lib  # noqa: F401  (fixture)

WORKER = textwrap.dedent(r'''
    import ctypes, os, sys, threading, time, traceback
    sys.path.insert(0, sys.argv[1])
    import distributedfft_b200.api as api
    api.LIB_PATH = sys.argv[2]
    api._lib = None
    import distributedfft_b200 as dfft
    L = dfft.lib()
    L.fakecuda_launch_setup.restype = ctypes.c_longlong
    L.fakecuda_launch_setup.argtypes = [ctypes.c_char_p, ctypes.c_longlong]

    def alloc(nbytes):
        return dfft.fft_mpi_alloc_local_memory((nbytes + 15) // 16, dfft.ALLOC_DEV)

    n0, n1, n2, P = 16, 512, 512, 2
    comm = dfft.LocalComm(P)
    errs, masks = [], [0] * P
    def worker(p):
        try:
            assert L.cudaSetDevice(p) == 0
            mc = dfft.getMaxDataCount(n0, n1, n2, P, p == P - 1)
            a = dfft.fft_mpi_alloc_local_memory(mc, dfft.ALLOC_DEV, dfft.FLOAT)
            b = dfft.fft_mpi_alloc_local_memory(mc, dfft.ALLOC_DEV, dfft.FLOAT)
            plan = dfft.fft_mpi_plan_dft_c2c_3d(n0, n1, n2, a, b, comm, p, P, dfft.FORWARD, dfft.FLOAT, dfft.EXCHANGE_P2P | dfft.NO_FUSE)
            for _ in range(2):
                plan.execute()
            plan.synchronize()
            masks[p] = plan.tma_mask
            plan.destroy()
            L.dfft_free_local(a, dfft.ALLOC_DEV); L.dfft_free_local(b, dfft.ALLOC_DEV)
        except Exception:
            errs.append(traceback.format_exc())
    th = [threading.Thread(target=worker, args=(p,), daemon=True) for p in range(P)]
    [t.start() for t in th]
    deadline = time.time() + 120
    while any(t.is_alive() for t in th) and not errs and time.time() < deadline:
        time.sleep(0.05)
    if errs or any(t.is_alive() for t in th):   # a device-thread that failed leaves its peer waiting for it
        print("\n".join(errs) or "device-threads did not finish", flush=True)
        os._exit(1)
    comm.destroy()
    assert all(masks), ("the plans ran no TMA kernel", masks)

    nx, ny, nz, batch = 16, 16, 8, 3
    d = alloc(nx * ny * nz * batch * 16)
    plan = dfft.LinesPlan(three_d=(nx, ny, nz, batch))
    for direction in (dfft.FORWARD, dfft.BACKWARD):
        plan.execute(d, direction)
    plan.synchronize(); plan.destroy()
    n, images = 32, 4
    i, o, m = alloc(n * n * images * 16), alloc(n * n * images * 16), alloc(n * n * 16)
    plan = dfft.LinesConvolvePlan(two_d=(n, n, images))
    for _ in range(2):
        plan.execute(i, o, m)
    plan.synchronize(); plan.destroy()
    for x in (d, i, o, m):
        L.dfft_free_local(x, dfft.ALLOC_DEV)

    need = L.fakecuda_launch_setup(None, 0)
    buf = ctypes.create_string_buffer(int(need))
    L.fakecuda_launch_setup(buf, need)
    print("SETUP")
    print(buf.value.decode(), end="")
''')


def test_each_pass_kernel_is_set_up_once_per_device(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, FAKECUDA_TMA="1")
    for k in ("DFFT_TMA", "DFFT_GENERIC", "DFFT_NO_PLANE", "DFFT_FORCE_PLANE"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    lines = r.stdout.split("SETUP\n", 1)[1].splitlines()
    launched = {}   # (device, mangled name) -> (opt-ins, occupancy queries, kernel)
    for line in lines:
        dev, attr, occ, launches, name = line.split(" ", 4)
        k = re.search(r"\d(fft_\w*?kernel)", name)
        if k and int(launches) > 0:
            launched[int(dev), name] = (int(attr), int(occ), k.group(1))
    bad = ["device %d %s: %d opt-ins, want 1" % (d, kern, a) for (d, _), (a, _, kern) in launched.items() if a != 1]
    bad += ["device %d %s: %d occupancy queries, want at most 1" % (d, kern, q) for (d, _), (_, q, kern) in launched.items()
            if q > 1 and not kern.startswith("fft_generic_")]
    assert not bad, "\n".join(bad)
    kinds = {(d, kern) for (d, _), (_, _, kern) in launched.items()}
    assert {(0, "fft_tma_pass_kernel"), (1, "fft_tma_pass_kernel"), (0, "fft_plane_kernel"), (0, "fft_plane_conv_kernel")} <= kinds, sorted(kinds)
