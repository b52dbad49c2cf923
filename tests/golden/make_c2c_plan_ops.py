"""Writes tests/golden/c2c_plan_ops.json: the passes (dfft_debug_plan_ops) that a set of fixed complex-to-complex DRY_RUN
plans record, per device.  The file pins the C2C schedules: tests/test_r2c_dry_run.py checks that the library still records
exactly these passes, so a change that adds a transform type cannot alter the C2C launches or their arguments unnoticed.

    python tests/golden/make_c2c_plan_ops.py

Regenerate only when a C2C schedule is meant to change, and say so in that change."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import distributedfft_b200 as dfft  # noqa: E402

OUT = os.path.join(HERE, "c2c_plan_ops.json")
# environment variables that change a plan's schedule; the capture and the check run without them
SCHEDULE_ENV = ("DFFT_FUSE", "DFFT_LAG", "DFFT_OVERLAP", "DFFT_PIPELINE", "DFFT_PIPELINE_BWD", "DFFT_PARTS", "DFFT_PIPE_MODE",
                "DFFT_EXCHANGE", "DFFT_GENERIC", "DFFT_VARIANT", "DFFT_SIGNAL_KERNELS")

# (P, n0, n1, n2, flags name): P = 1, 3 (uneven split) and 8; P2P and NCCL; fused (square planes) and unfused
CASES = [
    (1, 16, 16, 16, "default"), (1, 16, 16, 16, "FORCE_FUSE"), (1, 12, 10, 24, "NO_FUSE"), (1, 12, 10, 24, "NATURAL_SPECTRUM"),
    (3, 10, 16, 16, "EXCHANGE_P2P"), (3, 10, 16, 16, "EXCHANGE_P2P|NO_FUSE"), (3, 10, 9, 24, "EXCHANGE_NCCL"),
    (8, 24, 16, 16, "EXCHANGE_P2P"), (8, 24, 16, 16, "EXCHANGE_P2P|NO_FUSE"), (8, 24, 16, 16, "EXCHANGE_NCCL"),
]


def flag_value(name):
    v = 0
    for part in name.split("|"):
        if part != "default":
            v |= getattr(dfft, part)
    return v


def fake(dev, buf):
    return ((dev + 1) << 44) | (buf << 40)


def record(P, n0, n1, n2, flags, direction):
    per_dev = []
    for d in range(P):
        p = dfft.fft_mpi_plan_dft_c2c_3d(n0, n1, n2, fake(d, 5), fake(d, 2), None, d, P, direction, dfft.DOUBLE, flag_value(flags) | dfft.DRY_RUN)
        p.execute()
        per_dev.append(p.recorded_ops())
        p.destroy()
    return per_dev


def key(P, n0, n1, n2, flags, direction):
    return f"P{P}_{n0}x{n1}x{n2}_{flags}_{'fwd' if direction == dfft.FORWARD else 'bwd'}"


def main():
    for v in SCHEDULE_ENV:
        os.environ.pop(v, None)
    out = {}
    for P, n0, n1, n2, flags in CASES:
        for direction in (dfft.FORWARD, dfft.BACKWARD):
            out[key(P, n0, n1, n2, flags, direction)] = record(P, n0, n1, n2, flags, direction)
    with open(OUT, "w") as f:
        json.dump(out, f, indent=None, sort_keys=True)
        f.write("\n")
    print("wrote", OUT, len(out), "plans")


if __name__ == "__main__":
    main()
