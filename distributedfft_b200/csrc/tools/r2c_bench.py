#!/usr/bin/env python
"""R2C forward against the C2C forward on the same real data, one GPU (developer tool).

    python distributedfft_b200/csrc/tools/r2c_bench.py [--n 512] [--steps 50] [--rounds 3] [--float]

Both plans are created once.  The C2C plan gets the real cube widened to complex (imaginary parts 0), its default flags (fused
TMA t0 where that exists).  Each round times `steps` executes of one plan with CUDA events on the plan's stream, then the other,
alternating R2C and C2C, after a few untimed warm-up executes.  Prints one JSON object: card name, power limit and SM clock
(nvidia-smi, read-only query) before and after, ms per step of every round, and the per-pass times (Z, Y, X) of each plan's
last execute.  The spectra are compared too: the R2C spectrum must equal the first n2/2+1 z-columns of the C2C spectrum."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim, clk = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock": clk}
    except Exception as exc:   # the numbers still stand; the record says why the card state is missing
        return {"error": str(exc)}


def time_steps(torch, plan, steps):
    st = torch.cuda.ExternalStream(plan.stream)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(steps):
        plan.execute()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--float", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    import distributedfft_b200 as dfft

    n = args.n
    prec = dfft.FLOAT if args.float else dfft.DOUBLE
    rdt, cdt = (torch.float32, torch.complex64) if args.float else (torch.float64, torch.complex128)
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(1)
    real = torch.randn(n, n, n, dtype=rdt, device="cuda", generator=gen)
    rc, cc = dfft.local_size_r2c_3d(n, n, n, 1, 0)
    spec = torch.empty(cc, dtype=cdt, device="cuda")
    r2c = dfft.fft_mpi_plan_dft_r2c_3d(n, n, n, real.data_ptr(), spec.data_ptr(), None, 0, 1, dfft.FORWARD, prec)
    cin = real.to(cdt).reshape(-1)
    cout = torch.empty(n ** 3, dtype=cdt, device="cuda")
    c2c = dfft.fft_mpi_plan_dft_c2c_3d(n, n, n, cin.data_ptr(), cout.data_ptr(), None, 0, 1, dfft.FORWARD, prec)
    del cin
    state_before = gpu_state()
    for p in (r2c, c2c):
        for _ in range(args.warmup):
            p.execute()
        p.synchronize()
    rounds = []
    for _ in range(args.rounds):
        rounds.append({"r2c_ms": time_steps(torch, r2c, args.steps), "c2c_ms": time_steps(torch, c2c, args.steps)})
    r2c.execute(); r2c.synchronize()
    c2c.execute(); c2c.synchronize()
    h = n // 2 + 1
    full = cout.reshape(n, n, n)[:, :h, :]                      # [y][z][x], z cut to n/2+1
    diff = (spec.reshape(n, h, n) - full).abs().max().item() / full.abs().max().item()
    res = {
        "shape": [n, n, n], "precision": "float" if args.float else "double", "steps": args.steps, "rounds": rounds,
        "r2c_ms_median": float(np.median([r["r2c_ms"] for r in rounds])), "c2c_ms_median": float(np.median([r["c2c_ms"] for r in rounds])),
        "r2c_pass_ms": r2c.pass_timings(), "c2c_pass_ms": c2c.pass_timings(), "r2c_t": r2c.timings(), "c2c_t": c2c.timings(),
        "c2c_fused": c2c.fused, "c2c_tma_mask": c2c.tma_mask, "r2c_tma_mask": r2c.tma_mask,
        "r2c_vs_c2c_rel_max_diff": diff, "gpu_before": state_before, "gpu_after": gpu_state(),
    }
    r2c.destroy()
    c2c.destroy()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
