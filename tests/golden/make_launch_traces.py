"""Writes tests/golden/launch_traces.json: one SHA-256 per (plan, device-thread) of the ordered launch trace that non-dry plans
leave on the fake CUDA runtime (tests/fakecuda/fake_cudart.cpp, fakecuda_trace): every kernel launch with its device name,
grid, block, dynamic shared memory and stream, every event record and stream wait, every async copy and set, in issue order.
DRY_RUN records see neither the gate and signal kernels nor the event brackets; this trace does.
tests/test_launch_trace_fakecuda.py checks that the library still issues exactly these traces.

    python tests/golden/make_launch_traces.py [FAKE_LIB]              # rewrite the digests
    python tests/golden/make_launch_traces.py [FAKE_LIB] --show KEY   # print the full traces of the plans whose key contains KEY

FAKE_LIB defaults to distributedfft_b200/build/libdfft_fakecuda.so, which the fakecuda tests build.  Regenerate only when a
schedule is meant to change, and say so in that change."""
import hashlib
import json
import os
import subprocess
import sys
import textwrap

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "launch_traces.json")
FAKE_LIB = os.path.join(ROOT, "distributedfft_b200", "build", "libdfft_fakecuda.so")
SCHEDULE_ENV = ("DFFT_FUSE", "DFFT_LAG", "DFFT_OVERLAP", "DFFT_PIPELINE", "DFFT_PIPELINE_BWD", "DFFT_PARTS", "DFFT_PIPE_MODE",
                "DFFT_EXCHANGE", "DFFT_GENERIC", "DFFT_VARIANT", "DFFT_SIGNAL_KERNELS", "DFFT_TMA", "DFFT_PIPE_CAP",
                "DFFT_DEBUG_TIMELINE", "DFFT_NO_TMA")
# one worker process per runtime flavour: the TMA entry point is looked up once per process
FLAVOURS = {"notma": {}, "tma": {"FAKECUDA_TMA": "1"}, "tma2": {"FAKECUDA_TMA": "1", "DFFT_TMA": "2"}}

WORKER = textwrap.dedent(r'''
    import ctypes, json, os, sys, threading
    sys.path.insert(0, sys.argv[1])
    import distributedfft_b200.api as api
    api.LIB_PATH = sys.argv[2]
    api._lib = None
    import distributedfft_b200 as dfft
    L = dfft.lib()
    L.fakecuda_trace.restype = ctypes.c_longlong
    L.fakecuda_trace.argtypes = [ctypes.c_char_p, ctypes.c_longlong]
    tma = bool(os.environ.get("FAKECUDA_TMA"))

    def trace():
        n = L.fakecuda_trace(None, 0)
        buf = ctypes.create_string_buffer(int(n))
        L.fakecuda_trace(buf, n)
        return buf.value.decode().splitlines()

    def drive(kind, n0, n1, n2, P, flags, direction, precision, inplace=False, executes=2):
        comm = dfft.LocalComm(P) if P > 1 else None
        errs, out = [], [None] * P
        def worker(p):
            try:
                L.fakecuda_trace_reset()
                mc = dfft.getMaxDataCount(n0, n1, n2, P, p == P - 1)
                a = dfft.fft_mpi_alloc_local_memory(mc, dfft.ALLOC_DEV, precision)
                b = None if inplace else dfft.fft_mpi_alloc_local_memory(mc, dfft.ALLOC_DEV, precision)
                m = dfft.fft_mpi_alloc_local_memory(mc, dfft.ALLOC_DEV, precision)
                if kind == "c2c":
                    plan = dfft.fft_mpi_plan_dft_c2c_3d(n0, n1, n2, a, b, comm, p, P, direction, precision, flags)
                elif kind == "r2c":
                    plan = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, a, b, comm, p, P, direction, precision, flags)
                else:
                    plan = dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, a, b, comm, p, P, precision, flags, real=kind == "conv_r2c")
                for _ in range(executes):
                    if kind.startswith("conv"):
                        plan.execute_convolve(m)
                    else:
                        plan.execute()
                plan.synchronize()
                plan.timings(); plan.pass_timings()
                info = "launches %d fused %d parts %d chain %d tma_mask %d" % (plan.launches, plan.fused, plan.pipeline_parts,
                                                                              plan.pipeline_chain, plan.tma_mask)
                plan.destroy()
                out[p] = trace() + [info]
                for x in (a, b, m):
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
        return out

    F = {"default": 0}
    for name in ("NO_FUSE", "FORCE_FUSE", "SCALE_BACKWARD", "NATURAL_SPECTRUM", "FORCE_PIPELINE", "OVERLAP_X", "EXCHANGE_P2P"):
        F[name] = getattr(dfft, name)
    def flags_of(name):
        v = 0
        for part in name.split("|"):
            v |= F[part]
        return v

    cases = []
    kinds = ("c2c", "r2c", "conv_c2c", "conv_r2c")
    if tma:
        shapes = {1: [(8, 256, 256), (8, 512, 512)], 2: [(16, 512, 512)]}
        fusions = ("default", "NO_FUSE")
    else:
        shapes = {1: [(16, 16, 16), (12, 10, 24)], 2: [(16, 16, 16), (10, 12, 24)], 4: [(16, 16, 16), (10, 12, 24)]}
        fusions = ("default", "NO_FUSE", "FORCE_FUSE", "SCALE_BACKWARD")
    precs = {"f64": dfft.DOUBLE, "f32": dfft.FLOAT}
    for kind in kinds:
        dirs = (0,) if kind.startswith("conv") else (dfft.FORWARD, dfft.BACKWARD)
        for P, shs in shapes.items():
            for sh in shs:
                for fl in fusions:
                    name = fl if P == 1 else "EXCHANGE_P2P|" + fl if fl != "default" else "EXCHANGE_P2P"
                    for d in dirs:
                        for pn, prec in precs.items():
                            cases.append((kind, sh, P, name, d, pn, False))
    if not tma:
        for d in (dfft.FORWARD, dfft.BACKWARD):
            for kind in ("c2c", "r2c"):
                cases.append((kind, (12, 10, 24), 1, "NATURAL_SPECTRUM", d, "f64", False))
            cases.append(("c2c", (16, 16, 16), 1, "default", d, "f64", True))
            cases.append(("c2c", (10, 12, 24), 2, "EXCHANGE_P2P", d, "f64", True))
            for P in (2, 4):
                for sh in ((128, 128, 128), (8, 128, 128), (8, 12, 128)):
                    cases.append(("c2c", sh, P, "EXCHANGE_P2P|FORCE_PIPELINE", d, "f64", False))
                cases.append(("c2c", (64, 64, 64), P, "EXCHANGE_P2P|OVERLAP_X", d, "f64", False))
        cases.append(("conv_c2c", (16, 16, 16), 2, "EXCHANGE_P2P", 0, "f64", True))
        cases.append(("conv_r2c", (16, 16, 16), 1, "default", 0, "f32", True))
    result = {}
    for kind, sh, P, name, d, pn, inplace in cases:
        pipe_modes = (None, "streams") if "FORCE_PIPELINE" in name else (None,)
        for mode in pipe_modes:
            if mode: os.environ["DFFT_PIPE_MODE"] = mode
            key = "%s_P%d_%dx%dx%d_%s_%s" % (kind, P, sh[0], sh[1], sh[2], name, pn)
            if d: key += "_fwd" if d == dfft.FORWARD else "_bwd"
            if inplace: key += "_inplace"
            if mode: key += "_" + mode
            result[key] = drive(kind, *sh, P, flags_of(name), d, precs[pn], inplace)
            os.environ.pop("DFFT_PIPE_MODE", None)
    print(json.dumps(result))
''')


def traces(fake_lib, flavour):
    """{plan key: [trace lines of device-thread 0, 1, ...]} of one runtime flavour"""
    env = {k: v for k, v in os.environ.items() if k not in SCHEDULE_ENV and k != "FAKECUDA_TMA"}
    env.update(FLAVOURS[flavour])
    r = subprocess.run([sys.executable, "-c", WORKER, ROOT, fake_lib], capture_output=True, text=True, timeout=600, env=env)
    if r.returncode != 0:
        raise RuntimeError(r.stdout[-3000:] + r.stderr[-3000:])
    return {flavour + ":" + k: v for k, v in json.loads(r.stdout.splitlines()[-1]).items()}


def digest(lines):
    return hashlib.sha256("\n".join(lines).encode()).hexdigest()


def main(argv):
    show = None
    if "--show" in argv:
        i = argv.index("--show")
        show = argv[i + 1]
        argv = argv[:i] + argv[i + 2:]
    lib = argv[0] if argv else FAKE_LIB
    out = {}
    for flavour in FLAVOURS:
        for k, per_thread in traces(lib, flavour).items():
            if show is not None and show in k:
                for t, lines in enumerate(per_thread):
                    print("== %s thread %d" % (k, t))
                    print("\n".join(lines))
            out[k] = [digest(lines) for lines in per_thread]
    if show is not None:
        return
    with open(OUT, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", OUT, len(out), "plans")


if __name__ == "__main__":
    main(sys.argv[1:])
