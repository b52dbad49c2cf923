"""Writes tests/golden/plan_ops.json: one SHA-256 per DRY_RUN plan of the passes (dfft_debug_plan_ops) it records on every
device, for C2C, R2C and both convolve plans over 1, 2, 3 (uneven split) and 8 devices, P2P and NCCL, default / NO_FUSE /
FORCE_FUSE, both directions and both precisions, plus scaled, natural-spectrum, in-place, pipelined and overlapped C2C cases.
tests/test_plan_ops_golden.py checks that the library still records exactly these schedules.

    python tests/golden/make_plan_ops.py              # rewrite the digests
    python tests/golden/make_plan_ops.py KEY [KEY..]  # print the full records of these plans (to diff a mismatch)

The full records (several MB) are not stored.  Regenerate only when a schedule is meant to change, and say so in that change."""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import distributedfft_b200 as dfft  # noqa: E402

OUT = os.path.join(HERE, "plan_ops.json")
# environment variables that change a plan's schedule; the capture and the check run without them (DFFT_PIPE_MODE is set per case)
SCHEDULE_ENV = ("DFFT_FUSE", "DFFT_LAG", "DFFT_OVERLAP", "DFFT_PIPELINE", "DFFT_PIPELINE_BWD", "DFFT_PARTS", "DFFT_PIPE_MODE",
                "DFFT_EXCHANGE", "DFFT_GENERIC", "DFFT_VARIANT", "DFFT_SIGNAL_KERNELS")

KINDS = ("c2c", "r2c", "conv_c2c", "conv_r2c")
SHAPES = {1: (16, 16, 16), 2: (16, 16, 16), 3: (10, 16, 16), 8: (24, 16, 16)}   # square planes: fusion applies
MULT = 8


def fake(dev, buf):
    return ((dev + 1) << 44) | (buf << 40)


def flag_value(name):
    v = 0
    for part in name.split("|"):
        if part != "default":
            v |= getattr(dfft, part)
    return v


def cases():
    """(kind, P, n0, n1, n2, flags, direction or 0 for convolve, precision name, inplace, DFFT_PIPE_MODE)"""
    out = []
    for kind in KINDS:
        dirs = (0,) if kind.startswith("conv") else (dfft.FORWARD, dfft.BACKWARD)
        for P, shape in SHAPES.items():
            for xch in (("EXCHANGE_P2P",) if P == 1 else ("EXCHANGE_P2P", "EXCHANGE_NCCL")):
                for fuse in ("", "|NO_FUSE", "|FORCE_FUSE"):
                    for d in dirs:
                        for prec in ("f64", "f32"):
                            out.append((kind, P, *shape, xch + fuse, d, prec, False, None))
            for xch in (("EXCHANGE_P2P",) if P == 1 else ("EXCHANGE_P2P", "EXCHANGE_NCCL")):
                for d in dirs:
                    out.append((kind, P, *shape, xch + "|SCALE_BACKWARD", d, "f64", False, None))
        out.append((kind, 1, 12, 10, 24, "EXCHANGE_P2P", dirs[0], "f64", False, None))     # non-square planes, generic lengths
        if not kind.startswith("conv"):
            for d in dirs:
                out.append((kind, 1, 12, 10, 24, "NATURAL_SPECTRUM", d, "f64", False, None))
                out.append((kind, 1, 16, 16, 16, "NATURAL_SPECTRUM", d, "f32", False, None))
    for P in (1, 3):
        for xch in ("EXCHANGE_P2P", "EXCHANGE_NCCL") if P > 1 else ("EXCHANGE_P2P",):
            for d in (dfft.FORWARD, dfft.BACKWARD):
                out.append(("c2c", P, *SHAPES[P], xch, d, "f64", True, None))
    for kind in ("conv_c2c", "conv_r2c"):
        out.append((kind, 3, *SHAPES[3], "EXCHANGE_P2P", 0, "f64", True, None))
    # pipelined C2C: the kernel chain (cube, P2P forward), two streams (forced, and P2P / NCCL backward), fused and unfused part 0
    for P in (2, 4):
        for d in (dfft.FORWARD, dfft.BACKWARD):
            for shape in ((128, 128, 128), (8, 128, 128), (8, 12, 128)):
                for xch in ("EXCHANGE_P2P", "EXCHANGE_NCCL"):
                    for mode in (None, "streams"):
                        out.append(("c2c", P, *shape, xch + "|FORCE_PIPELINE", d, "f64", False, mode))
    # overlapped forward (one kernel for t0..t3), and the flag on a backward plan where it does nothing
    for P in (2, 3, 8):
        for d in (dfft.FORWARD, dfft.BACKWARD):
            out.append(("c2c", P, *SHAPES[P], "EXCHANGE_P2P|OVERLAP_X", d, "f64", False, None))
    out.append(("c2c", 4, 64, 64, 64, "EXCHANGE_P2P|OVERLAP_X", dfft.FORWARD, "f64", False, None))
    return out


def key(c):
    kind, P, n0, n1, n2, flags, d, prec, inplace, mode = c
    k = f"{kind}_P{P}_{n0}x{n1}x{n2}_{flags}_{prec}"
    if d:
        k += "_fwd" if d == dfft.FORWARD else "_bwd"
    if inplace:
        k += "_inplace"
    if mode:
        k += "_" + mode
    return k


def record(c):
    kind, P, n0, n1, n2, flags, d, prec, inplace, mode = c
    precision = dfft.DOUBLE if prec == "f64" else dfft.FLOAT
    fl = flag_value(flags) | dfft.DRY_RUN
    if mode:
        os.environ["DFFT_PIPE_MODE"] = mode
    try:
        per_dev = []
        for dev in range(P):
            out = None if inplace else fake(dev, 2)
            if kind == "c2c":
                p = dfft.fft_mpi_plan_dft_c2c_3d(n0, n1, n2, fake(dev, 5), out, None, dev, P, d, precision, fl)
            elif kind == "r2c":
                p = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, fake(dev, 5), out, None, dev, P, d, precision, fl)
            else:
                p = dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, fake(dev, 5), out, None, dev, P, precision, fl, real=kind == "conv_r2c")
            if kind.startswith("conv"):
                p.execute_convolve(fake(dev, MULT))
            else:
                p.execute()
            per_dev.append({"ops": p.recorded_ops(), "launches": p.launches, "fused": p.fused, "parts": p.pipeline_parts,
                            "chain": p.pipeline_chain})
            p.destroy()
        return per_dev
    finally:
        os.environ.pop("DFFT_PIPE_MODE", None)


def digest(per_dev):
    return hashlib.sha256(json.dumps(per_dev, sort_keys=True).encode()).hexdigest()


def main(argv):
    for v in SCHEDULE_ENV:
        os.environ.pop(v, None)
    by_key = {key(c): c for c in cases()}
    assert len(by_key) == len(cases()), "duplicate case keys"
    if argv:
        for k in argv:
            print(k)
            print(json.dumps(record(by_key[k]), indent=1, sort_keys=True))
        return
    out = {k: digest(record(c)) for k, c in by_key.items()}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", OUT, len(out), "plans")


if __name__ == "__main__":
    main(sys.argv[1:])
