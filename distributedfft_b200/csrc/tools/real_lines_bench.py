#!/usr/bin/env python
"""Real lines plans against C2C lines plans on the same data, one GPU (developer tool).

    python distributedfft_b200/csrc/tools/real_lines_bench.py [--steps 50] [--rounds 3] [--warmup 5] [--min-gib 1.0] [--case NAME]

For every case a RealLinesPlan and a C2C LinesPlan are created once; the C2C plan gets the same seeded real data widened to
complex (imaginary parts 0) and transforms it in place.  Each round times `steps` executes of each plan with CUDA events on the
plan's own stream, alternating real and C2C, forward then backward, after `warmup` untimed executes.  Line counts (1-D) and
batches (2-D) are raised until the real input is at least `--min-gib` GiB, so that the 50 MB L2 holds no meaningful share of it.
Before timing, the real forward result is compared with the first n/2+1 bins of the C2C result.

Prints one JSON object per case and a summary table: ms per step of each plan (median of the rounds), their ratio, and achieved
GB/s from the algorithmic bytes of one read and one write: E_r*n + E_c*(n/2+1) per real line, 2*E_c*n per complex line (E_r,
E_c: bytes of a real / complex element; 2-D plans count each row once, as if the transform moved the data once).  Card name,
power limit and SM clock (nvidia-smi, read-only query) are printed before and after."""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)

# name, precision ("d" / "f"), n (real axis), ny (0: 1-D), nominal batch (2-D; raised to reach the input size)
CASES = [
    ("1d-512", "d", 512, 0, 0), ("1d-1024", "d", 1024, 0, 0), ("1d-4096", "d", 4096, 0, 0),
    ("1d-360-gen", "d", 360, 0, 0), ("1d-480-gen", "d", 480, 0, 0),
    ("2d-1024x1024", "d", 1024, 1024, 16),
    ("1d-768-f32", "f", 768, 0, 0), ("2d-768x768-f32", "f", 768, 768, 16),
]


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim, clk = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock": clk}
    except Exception as exc:   # the numbers still stand; the record says why the card state is missing
        return {"error": str(exc)}


def time_steps(torch, stream, fn, steps):
    st = torch.cuda.ExternalStream(stream)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(steps):
        fn()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) / steps


def run_case(torch, np, dfft, case, args):
    name, p, n, ny, batch0 = case
    prec = dfft.FLOAT if p == "f" else dfft.DOUBLE
    rdt, cdt = (torch.float32, torch.complex64) if p == "f" else (torch.float64, torch.complex128)
    er = 4 if p == "f" else 8
    ec = 2 * er
    H = n // 2 + 1
    want = args.min_gib * 2 ** 30
    if ny:
        batch = max(batch0, math.ceil(want / (ny * n * er)))
        rows, real_kw, c2c_kw = ny * batch, {"two_d": (n, ny, batch)}, {"two_d": (n, ny, batch)}
    else:
        rows = math.ceil(want / (n * er))
        batch = 0
        real_kw = {"n": n, "nlines": rows}
        c2c_kw = {"n": n, "stride": 1, "nlines": rows, "inner": rows, "inner_dist": n, "outer_dist": 0}
    gen = torch.Generator(device="cuda").manual_seed(7)
    real = torch.randn(rows * n, dtype=rdt, device="cuda", generator=gen)
    spec = torch.empty(rows * H, dtype=cdt, device="cuda")
    back = torch.empty(rows * n, dtype=rdt, device="cuda")
    data = real.to(cdt)
    rp = dfft.RealLinesPlan(precision=prec, **real_kw)
    cp = dfft.LinesPlan(precision=prec, **c2c_kw)
    try:
        rp.execute(real.data_ptr(), spec.data_ptr(), dfft.FORWARD)
        rp.synchronize()
        cp.execute(data.data_ptr(), dfft.FORWARD)
        cp.synchronize()
        ref = data.reshape(rows, n)[:, :H] if not ny else data.reshape(batch, ny, n)[:, :, :H].reshape(rows, H)
        diff = ((spec.reshape(rows, H) - ref).abs().max() / ref.abs().max()).item()
        del ref
        jobs = {
            "real_fwd": (rp.stream, lambda: rp.execute(real.data_ptr(), spec.data_ptr(), dfft.FORWARD)),
            "c2c_fwd": (cp.stream, lambda: cp.execute(data.data_ptr(), dfft.FORWARD)),
            "real_bwd": (rp.stream, lambda: rp.execute(spec.data_ptr(), back.data_ptr(), dfft.BACKWARD)),
            "c2c_bwd": (cp.stream, lambda: cp.execute(data.data_ptr(), dfft.BACKWARD)),
        }
        for st, fn in jobs.values():
            for _ in range(args.warmup):
                fn()
            torch.cuda.ExternalStream(st).synchronize()
        rounds = []
        for _ in range(args.rounds):
            rounds.append({k: time_steps(torch, st, fn, args.steps) for k, (st, fn) in jobs.items()})
    finally:
        rp.destroy()
        cp.destroy()
    med = {k: float(np.median([r[k] for r in rounds])) for k in rounds[0]}
    real_bytes, c2c_bytes = rows * (er * n + ec * H), rows * 2 * ec * n
    res = {
        "case": name, "precision": "float" if p == "f" else "double", "n": n, "ny": ny, "batch": batch, "lines": rows,
        "real_input_gib": rows * n * er / 2 ** 30, "steps": args.steps, "rounds": rounds, "median_ms": med,
        "ratio_fwd": med["real_fwd"] / med["c2c_fwd"], "ratio_bwd": med["real_bwd"] / med["c2c_bwd"],
        "gbps": {"real_fwd": real_bytes / med["real_fwd"] / 1e6, "c2c_fwd": c2c_bytes / med["c2c_fwd"] / 1e6,
                 "real_bwd": real_bytes / med["real_bwd"] / 1e6, "c2c_bwd": c2c_bytes / med["c2c_bwd"] / 1e6},
        "real_vs_c2c_rel_max_diff": diff,
    }
    del real, spec, back, data
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-gib", type=float, default=1.0)
    ap.add_argument("--case", action="append", help="run only these cases (default: all)")
    args = ap.parse_args()
    import numpy as np
    import torch
    import distributedfft_b200 as dfft

    torch.cuda.set_device(0)
    before = gpu_state()
    print(json.dumps({"gpu_before": before}), flush=True)
    results = []
    for case in CASES:
        if args.case and case[0] not in args.case:
            continue
        r = run_case(torch, np, dfft, case, args)
        results.append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps({"gpu_after": gpu_state()}), flush=True)
    print("%-16s %7s %9s %9s %6s %8s %8s %9s %9s %6s %8s %8s" % ("case", "lines", "real_fwd", "c2c_fwd", "ratio", "GB/s_r", "GB/s_c",
                                                                  "real_bwd", "c2c_bwd", "ratio", "GB/s_r", "GB/s_c"))
    for r in results:
        m, g = r["median_ms"], r["gbps"]
        print("%-16s %7d %9.3f %9.3f %6.3f %8.0f %8.0f %9.3f %9.3f %6.3f %8.0f %8.0f" % (
            r["case"], r["lines"], m["real_fwd"], m["c2c_fwd"], r["ratio_fwd"], g["real_fwd"], g["c2c_fwd"],
            m["real_bwd"], m["c2c_bwd"], r["ratio_bwd"], g["real_bwd"], g["c2c_bwd"]))


if __name__ == "__main__":
    main()
