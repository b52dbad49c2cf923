#!/usr/bin/env python
"""Batched 3-D lines plans: the plane kernel against the separate passes, one GPU (developer tool).

    python distributedfft_b200/csrc/tools/lines3d_bench.py [--steps 50] [--rounds 3] [--warmup 5] [--case NAME]

For every case three arms get the same seeded data: the plan created under DFFT_FORCE_PLANE=1 (LinesPlan(three_d=...) running the
X and Y passes as one fft_plane_kernel launch wherever one is instantiated, on by default or not), the same plan created under DFFT_NO_PLANE=1 (three
separate passes), and torch.fft.fftn over the last three axes (cuFFT; context only).  Real cases run RealLinesPlan(three_d=...)
in both plan arms (the real plans never use the plane kernel) and torch.fft.rfftn / irfftn.  Each round times `steps` executes
of each arm with CUDA events on the arm's own stream, arms alternating, forward then backward, after `warmup` untimed executes.
Before timing, one forward and one backward of the two plan arms from the same input are compared with np.array_equal.

Prints one JSON object per case and a summary table: ms per step (median of the rounds), the plane / passes ratio, and
algorithmic GB/s = one read and one write of the data per transform (C2C: 2*E*V; real: E_r*V + E_c*V_half) over the time; the
HBM sweeps each arm makes are listed beside them (C2C: 4*E*V with the plane kernel, 6*E*V without).  Card name, power limit and
SM clock (nvidia-smi, read-only query) are printed before and after."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)

# name, precision ("d" / "f"), (nx, ny, nz, batch), real
CASES = [
    ("64^3x256", "d", (64, 64, 64, 256), False), ("32^3x2048", "d", (32, 32, 32, 2048), False),
    ("16^3x16384", "d", (16, 16, 16, 16384), False),
    ("64^3x512-f32", "f", (64, 64, 64, 512), False), ("32^3x4096-f32", "f", (32, 32, 32, 4096), False),
    ("16^3x32768-f32", "f", (16, 16, 16, 32768), False),
    ("48^3x512", "d", (48, 48, 48, 512), False),
    ("real-64^3x256", "d", (64, 64, 64, 256), True),
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
    st = torch.cuda.ExternalStream(stream) if stream is not None else torch.cuda.current_stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    with torch.cuda.stream(st):
        for _ in range(steps):
            fn()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) / steps


def make_plan(dfft, shape, prec, real, no_plane):
    """no_plane: DFFT_NO_PLANE=1; else DFFT_FORCE_PLANE=1, so that an instantiation that is off by default is still measured"""
    var = "DFFT_NO_PLANE" if no_plane else "DFFT_FORCE_PLANE"
    os.environ[var] = "1"
    try:
        return dfft.RealLinesPlan(three_d=shape, precision=prec) if real else dfft.LinesPlan(three_d=shape, precision=prec)
    finally:
        os.environ.pop(var, None)


def run_case(torch, np, dfft, case, args):
    name, p, shape, real = case
    nx, ny, nz, batch = shape
    prec = dfft.FLOAT if p == "f" else dfft.DOUBLE
    rdt, cdt = (torch.float32, torch.complex64) if p == "f" else (torch.float64, torch.complex128)
    er = 4 if p == "f" else 8
    ec = 2 * er
    H = nx // 2 + 1
    V = nx * ny * nz * batch
    Vh = ny * nz * batch * H
    gen = torch.Generator(device="cuda").manual_seed(7)
    dims = (-3, -2, -1)
    plans = {"plane": make_plan(dfft, shape, prec, real, False), "passes": make_plan(dfft, shape, prec, real, True)}
    try:
        if not real:
            src = torch.randn(V, dtype=cdt, device="cuda", generator=gen)
            bufs = {k: src.clone() for k in plans}
            tin = src.reshape(batch, nz, ny, nx)
            tout = torch.empty_like(tin)
            # equality check: forward then backward of each plan arm from the same input
            for k, pl in plans.items():
                pl.execute(bufs[k].data_ptr(), dfft.FORWARD)
                pl.synchronize()
            eq_fwd = bool(torch.equal(bufs["plane"], bufs["passes"]))
            for k, pl in plans.items():
                pl.execute(bufs[k].data_ptr(), dfft.BACKWARD)
                pl.synchronize()
            eq_bwd = bool(torch.equal(bufs["plane"], bufs["passes"]))
            jobs = {}
            for d, dn in ((dfft.FORWARD, "fwd"), (dfft.BACKWARD, "bwd")):
                for k, pl in plans.items():
                    jobs[f"{k}_{dn}"] = (pl.stream, (lambda pl=pl, b=bufs[k], d=d: pl.execute(b.data_ptr(), d)))
                fn = torch.fft.fftn if d == dfft.FORWARD else torch.fft.ifftn
                jobs[f"torch_{dn}"] = (None, (lambda fn=fn: fn(tin, dim=dims, out=tout)))
            alg = 2 * ec * V
        else:
            x = torch.randn(V, dtype=rdt, device="cuda", generator=gen)
            spec = {k: torch.empty(Vh, dtype=cdt, device="cuda") for k in plans}
            back = {k: torch.empty(V, dtype=rdt, device="cuda") for k in plans}
            for k, pl in plans.items():
                pl.execute(x.data_ptr(), spec[k].data_ptr(), dfft.FORWARD)
                pl.execute(spec[k].data_ptr(), back[k].data_ptr(), dfft.BACKWARD)
                pl.synchronize()
            eq_fwd = bool(torch.equal(spec["plane"], spec["passes"]))
            eq_bwd = bool(torch.equal(back["plane"], back["passes"]))
            xin = x.reshape(batch, nz, ny, nx)
            sout = torch.empty(batch, nz, ny, H, dtype=cdt, device="cuda")
            bout = torch.empty_like(xin)
            jobs = {}
            for k, pl in plans.items():
                jobs[f"{k}_fwd"] = (pl.stream, (lambda pl=pl, k=k: pl.execute(x.data_ptr(), spec[k].data_ptr(), dfft.FORWARD)))
            jobs["torch_fwd"] = (None, lambda: torch.fft.rfftn(xin, dim=dims, out=sout))
            for k, pl in plans.items():
                jobs[f"{k}_bwd"] = (pl.stream, (lambda pl=pl, k=k: pl.execute(spec[k].data_ptr(), back[k].data_ptr(), dfft.BACKWARD)))
            jobs["torch_bwd"] = (None, lambda: torch.fft.irfftn(sout, s=(nz, ny, nx), dim=dims, out=bout))
            alg = er * V + ec * Vh
        for st, fn in jobs.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        rounds = []
        for _ in range(args.rounds):
            rounds.append({k: time_steps(torch, st, fn, args.steps) for k, (st, fn) in jobs.items()})
        torch.cuda.synchronize()
    finally:
        for pl in plans.values():
            pl.destroy()
    med = {k: float(np.median([r[k] for r in rounds])) for k in rounds[0]}
    plane_on = not real and any(o["op"] == "XY_PLANE" for o in dfft.lines_3d_ops(nx, ny, nz, batch, dfft.FORWARD, prec))   # by default
    res = {
        "case": name, "precision": "float" if p == "f" else "double", "shape": list(shape), "real": real,
        "gib": (V * (er if real else ec)) / 2 ** 30, "plane_kernel_default": plane_on, "steps": args.steps, "rounds": rounds,
        "median_ms": med, "ratio_fwd": med["plane_fwd"] / med["passes_fwd"], "ratio_bwd": med["plane_bwd"] / med["passes_bwd"],
        "alg_gbps": {k: alg / v / 1e6 for k, v in med.items()},
        "hbm_sweeps": {"plane": 2 if plane_on else 3, "passes": 3},
        "array_equal_plane_vs_passes": {"fwd": eq_fwd, "bwd": eq_bwd},
    }
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--case", action="append", help="run only these cases (default: all)")
    args = ap.parse_args()
    import numpy as np
    import torch
    import distributedfft_b200 as dfft

    torch.cuda.set_device(0)
    os.environ.pop("DFFT_NO_PLANE", None)
    print(json.dumps({"gpu_before": gpu_state()}), flush=True)
    results = []
    for case in CASES:
        if args.case and case[0] not in args.case:
            continue
        r = run_case(torch, np, dfft, case, args)
        results.append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps({"gpu_after": gpu_state()}), flush=True)
    print("%-16s %5s %9s %9s %9s %6s %7s %7s %9s %9s %9s %6s %6s" % (
        "case", "plane", "plane_f", "passes_f", "torch_f", "ratio", "GB/s_p", "GB/s_s", "plane_b", "passes_b", "torch_b", "ratio", "equal"))
    for r in results:
        m, g = r["median_ms"], r["alg_gbps"]
        print("%-16s %5s %9.3f %9.3f %9.3f %6.3f %7.0f %7.0f %9.3f %9.3f %9.3f %6.3f %6s" % (
            r["case"], "on" if r["plane_kernel_default"] else "off", m["plane_fwd"], m["passes_fwd"], m["torch_fwd"], r["ratio_fwd"],
            g["plane_fwd"], g["passes_fwd"], m["plane_bwd"], m["passes_bwd"], m["torch_bwd"], r["ratio_bwd"],
            all(r["array_equal_plane_vs_passes"].values())))


if __name__ == "__main__":
    main()
