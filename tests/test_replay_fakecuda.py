"""CPU test of the one-GPU replay of the multi-device schedules (tests/gpu_replay.py, test hook dfft_debug_launch_op) on the
fake CUDA runtime of test_control_flow_fakecuda.py (device memory = host memory, launches = counted no-ops).

The player drives every schedule test_gpu_chunked_replay.py replays -- P2P fused and NO_FUSE, NCCL, the stream-pipelined parts,
the fused t0 on square planes, convolve -- through the CPU footprint check and the hook; every record becomes exactly one
launch of the kernel its kind names (a fused pair one launch of the two-role kernel).  Every rejection of the hook comes back
as its code, and two mutations of the records (a chunk base shifted by a row, a C of another configuration) are caught before
anything is launched."""
import os
import subprocess
import sys
import textwrap

from test_control_flow_fakecuda import ROOT, fake_lib  # noqa: F401  (fixture)

WORKER = textwrap.dedent(r'''
    import copy, ctypes, os, sys
    sys.path.insert(0, sys.argv[1])
    sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
    import distributedfft_b200.api as api
    api.LIB_PATH = sys.argv[2]
    api._lib = None
    import numpy as np
    import distributedfft_b200 as dfft
    from oracle import SlabGeometry
    from gpu_replay import MULT, HostMemory, Replay, launch_units
    from test_dry_run import BUF1, IN, dry_ops, fake
    L = dfft.lib()
    L.fakecuda_launches.restype = ctypes.c_longlong
    L.fakecuda_trace.restype = ctypes.c_longlong
    L.fakecuda_trace.argtypes = [ctypes.c_char_p, ctypes.c_longlong]
    P2P, NCCL, NO_FUSE, NO_TMA, PIPE = dfft.EXCHANGE_P2P, dfft.EXCHANGE_NCCL, dfft.NO_FUSE, dfft.NO_TMA, dfft.FORCE_PIPELINE
    KERNEL = {"Z": "fft_tile_kernel", "Y": "fft_tile_kernel", "Y_CO": "fft_tile_kernel", "Y_CI": "fft_tile_kernel",
              "XF": "fft_tile_kernel", "XB": "fft_tile_kernel", "XB_CO": "fft_tile_kernel", "XCONV": "fft_conv_kernel",
              "XCONV_CO": "fft_conv_kernel", "fusedZ": "fft_fused2_kernel", "fusedY": "fft_fused2_kernel"}
    seen = set()

    def trace():
        n = L.fakecuda_trace(None, 0)
        buf = ctypes.create_string_buffer(int(n) + 1)
        L.fakecuda_trace(buf, n + 1)
        return [ln.split()[1] for ln in buf.value.decode().splitlines() if ln.startswith("launch ")]

    def inputs(g, direction, prec, inplace=False):
        npdt = np.complex128 if prec == dfft.DOUBLE else np.complex64
        cnt = [g.in_count(d) if direction == dfft.FORWARD else g.out_count(d) for d in range(g.P)]
        init = {(d, BUF1): np.ones(cnt[d], dtype=npdt) for d in range(g.P)}
        if inplace:
            init.update({(d, IN): np.ones(cnt[d], dtype=npdt) for d in range(g.P)})
        return init

    def play(g, ops, prec, init, nphases=2):
        L.fakecuda_trace_reset()
        before = L.fakecuda_launches()
        rep = Replay(g, ops, prec, init, nphases, mem=HostMemory())
        n = rep.run()
        units = [u for u in launch_units(ops, nphases) if u[1]["op"] != "alltoall"]
        assert n == len(units) == L.fakecuda_launches() - before, (n, len(units))
        names = trace()
        assert len(names) == n
        for (d, op, second), kname in zip(units, names):
            assert KERNEL[op["op"]] in kname or (KERNEL[op["op"]] == "fft_tile_kernel" and "fft_generic_kernel" in kname), (op["op"], kname)
            assert (second is not None) == (op["op"] in ("fusedZ", "fusedY"))
            seen.add(op["op"] if second is None else ("FK_ZY_CO" if "co" in second else "FK_ZY") if op["op"] == "fusedZ"
                     else ("FK_YZ_CI" if "ci" in op else "FK_YZ"))
        return rep

    def c2c(shape, P, direction, flags, prec=dfft.DOUBLE, inplace=False):
        g = SlabGeometry(*shape, P)
        ops, _ = dry_ops(*shape, P, direction, flags | NO_TMA, prec, inplace)
        return play(g, ops, prec, inputs(g, direction, prec, inplace))

    def conv(shape, P, flags, prec=dfft.DOUBLE):
        g = SlabGeometry(*shape, P)
        plans = [dfft.fft_mpi_plan_dft_convolve_3d(*shape, fake(d, IN), fake(d, 2), None, d, P, prec, flags | NO_TMA | dfft.DRY_RUN) for d in range(P)]
        ops = []
        for d, p in enumerate(plans):
            p.execute_convolve(fake(d, MULT))
            ops.append(p.recorded_ops())
            p.destroy()
        init = inputs(g, dfft.FORWARD, prec)
        npdt = np.complex128 if prec == dfft.DOUBLE else np.complex64
        init.update({(d, MULT): np.ones(g.out_count(d), dtype=npdt) for d in range(P)})
        return play(g, ops, prec, init, 4)

    for prec in (dfft.DOUBLE, dfft.FLOAT):
        for direction in (dfft.FORWARD, dfft.BACKWARD):
            for P in (2, 3):
                for flags in (P2P, P2P | NO_FUSE, NCCL):
                    c2c((9, 16, 10), P, direction, flags, prec, inplace=P == 3)
                    c2c((16, 9, 10), P, direction, flags, prec)
                    c2c((P, 64, 64), P, direction, flags | dfft.SCALE_BACKWARD, prec)
            for var, val, shape, P, flags in ((None, None, (8, 128, 128), 2, P2P), ("DFFT_PARTS", "2", (64, 64, 64), 2, P2P),
                                              ("DFFT_PIPE_MODE", "streams", (6, 64, 64), 3, P2P), (None, None, (8, 16, 128), 2, NCCL)):
                if var:
                    os.environ[var] = val
                c2c(shape, P, direction, flags | PIPE, prec)
                if var:
                    del os.environ[var]
        for P, mode in ((2, P2P), (3, P2P), (3, NCCL), (2, P2P | NO_FUSE)):
            conv((16, 16, 16), P, mode, prec)
            conv((12, 10, 9), P, mode, prec)
    want = {"Z", "Y_CO", "Y_CI", "XF", "XB", "XB_CO", "FK_ZY_CO", "FK_YZ_CI", "XCONV_CO", "XCONV"}
    assert want <= seen, want - seen

    # rejections of the hook, each with its code
    g = SlabGeometry(9, 16, 10, 2)
    ops, _ = dry_ops(9, 16, 10, 2, dfft.FORWARD, P2P | NO_TMA)
    rep = Replay(g, ops, dfft.DOUBLE, inputs(g, dfft.FORWARD, dfft.DOUBLE), mem=HostMemory())
    yco = rep.device_record(next(op for op in ops[0] if op["op"] == "Y_CO"))
    z = rep.device_record(next(op for op in ops[0] if op["op"] == "Z"))
    assert dfft.debug_launch_op(yco, dfft.DOUBLE) == 0 and dfft.debug_launch_op(z, dfft.DOUBLE) == 0
    def bad(**kw):
        r = copy.deepcopy(kw.pop("rec", yco))
        for k, v in kw.items():
            r[k] = v
        return r
    EINVAL = -1
    assert dfft.debug_launch_op(bad(op="Q"), dfft.DOUBLE) == EINVAL                      # unknown op
    for o in ("Z_R2C", "XY_PLANE", "XY_PLANE_CONV", "LINE_CONV", "LINE_CONV_R2C"):
        assert dfft.debug_launch_op(bad(op=o), dfft.DOUBLE) == EINVAL                    # a real-data or lines-engine record
    for o in ("ovlZ", "ovlY", "ovlX"):
        assert dfft.debug_launch_op(bad(op=o), dfft.DOUBLE) == EINVAL                    # single-kernel forward
    assert dfft.debug_launch_op(yco, 2) == EINVAL and dfft.debug_launch_op(yco, -1) == EINVAL   # precision
    assert dfft.debug_launch_op(bad(C=yco["C"] * 2), dfft.DOUBLE) == EINVAL             # not the entry's p_C
    assert dfft.debug_launch_op(bad(rec=z, C=z["C"] + 1), dfft.DOUBLE) == EINVAL        # not z_C
    assert dfft.debug_launch_op(bad(rec=z, **{"in": None}), dfft.DOUBLE) == EINVAL     # null pointers
    assert dfft.debug_launch_op(bad(rec=z, out=None), dfft.DOUBLE) == EINVAL
    nul = copy.deepcopy(yco); nul["co"]["cptr"][1] = None
    assert dfft.debug_launch_op(nul, dfft.DOUBLE) == EINVAL
    noch = copy.deepcopy(yco); del noch["co"]
    assert dfft.debug_launch_op(noch, dfft.DOUBLE) == EINVAL                               # Y_CO without its chunk table
    extra = copy.deepcopy(z); extra["co"] = yco["co"]
    assert dfft.debug_launch_op(extra, dfft.DOUBLE) == EINVAL                              # Z with one
    assert dfft.debug_launch_op(bad(G=yco["G"] + 1), dfft.DOUBLE) == EINVAL             # tiling inconsistent with W
    assert dfft.debug_launch_op(bad(rec=z, ntiles=z["ntiles"] + 1, G=max(2, z["G"])), dfft.DOUBLE) == EINVAL
    conv_ops = []
    for d in range(2):
        p = dfft.fft_mpi_plan_dft_convolve_3d(16, 16, 16, fake(d, IN), fake(d, 2), None, d, 2, dfft.DOUBLE, P2P | NO_TMA | dfft.DRY_RUN)
        p.execute_convolve(fake(d, MULT)); conv_ops.append(p.recorded_ops()); p.destroy()
    gc = SlabGeometry(16, 16, 16, 2)
    initc = inputs(gc, dfft.FORWARD, dfft.DOUBLE)
    initc.update({(d, MULT): np.ones(gc.out_count(d), dtype=np.complex128) for d in range(2)})
    repc = Replay(gc, conv_ops, dfft.DOUBLE, initc, 4, mem=HostMemory())
    xc = repc.device_record(next(op for op in conv_ops[0] if op["op"] == "XCONV_CO"))
    assert dfft.debug_launch_op(xc, dfft.DOUBLE) == 0
    assert dfft.debug_launch_op(bad(rec=xc, mult=None), dfft.DOUBLE) == EINVAL         # convolution without its multiplier
    fz = repc.device_record(next(op for op in conv_ops[0] if op["op"] == "fusedZ"))
    fy = repc.device_record(next(op for op in conv_ops[0] if op["op"] == "fusedY"))
    assert dfft.debug_launch_op(fz, dfft.DOUBLE, fy) == 0
    assert dfft.debug_launch_op(fz, dfft.DOUBLE) == EINVAL                                 # a fused role alone
    assert dfft.debug_launch_op(fz, dfft.DOUBLE, fz) == EINVAL                             # two Z roles
    assert dfft.debug_launch_op(bad(rec=fz, C=fy["C"] * 2), dfft.DOUBLE, fy) == EINVAL  # not f_zCp
    assert dfft.debug_launch_op(fz, dfft.DOUBLE, bad(rec=fy, C=fy["C"] * 2)) == EINVAL  # not the peer-store p_C
    assert dfft.debug_launch_op(z, dfft.DOUBLE, z) == EINVAL                               # a plain kind takes one record

    # mutations of the records are caught before any launch
    def mutated(fn):
        ops, _ = dry_ops(9, 16, 10, 2, dfft.FORWARD, P2P | NO_TMA)
        fn(ops)
        before = L.fakecuda_launches()
        try:
            Replay(g, ops, dfft.DOUBLE, inputs(g, dfft.FORWARD, dfft.DOUBLE), mem=HostMemory()).run()
        except AssertionError:
            return L.fakecuda_launches() - before
        raise SystemExit("mutation not caught: " + fn.__name__)
    def shifted_cptr(ops):
        next(op for op in ops[1] if op["op"] == "Y_CO")["co"]["cptr"][0] += 16 * 10      # device 1's rows in device 0 start a row late
    def wrong_configuration(ops):
        y = next(op for op in ops[0] if op["op"] == "Y_CO")
        yci, _ = dry_ops(9, 16, 10, 2, dfft.BACKWARD, P2P | NO_TMA)
        c = next(op for op in yci[0] if op["op"] == "Y_CI")["C"]                      # the local configuration's s_C
        planes = y["ntiles"] // y["G"]
        y["C"] = c if c != y["C"] else 2 * y["C"]
        y["G"] = -(-y["W"] // y["C"]); y["ntiles"] = planes * y["G"]
    assert mutated(shifted_cptr) == 0
    assert mutated(wrong_configuration) <= 1          # the Z pass of device 0 may have run; the Y_CO record is refused
    print("replay fakecuda ok", sorted(seen))
''')


def test_replay_player_on_a_fake_runtime(fake_lib, tmp_path):  # noqa: F811
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "replay fakecuda ok" in r.stdout
