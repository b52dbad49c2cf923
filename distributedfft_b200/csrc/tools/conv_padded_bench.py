#!/usr/bin/env python
"""Zero-padded batched 1-D convolution, out[l] = ifft(fft(in[l], n) * m)[:out_len]: the padded convolve lines plan against the
sequence it replaces and against torch, one GPU (developer tool).

    python distributedfft_b200/csrc/tools/conv_padded_bench.py [--seconds 1.0] [--warmup 5] [--case NAME]

Arms, on the same seeded data (nlines lines of in_len points, one shared multiplier of n points):
  plan      LinesConvolvePlan(one_d=(n, nlines), padded=(in_len, out_len)), out of place
  composed  torch pad to n, LinesPlan forward in place, torch multiply, LinesPlan backward, slice copied to a dense output
            (all on the lines plan's stream)
  torch     torch.fft.ifft(torch.fft.fft(a, n=n) * m)[..., :out_len] (cuFFT; the slice is a view)
Before timing, the plan's output is compared with both (rel_l2).  Each arm runs `warmup` untimed steps, then enough steps to fill
about `seconds` (CUDA events on the arm's stream).  nlines is chosen so that the input holds about 1 GiB.

Byte model (E = bytes per complex element, per line; M = the multiplier, read once per tile):
  plan, short path (n with a tuned kernel)    (in_len + out_len) E
  plan, long path (four-step, three passes)   (in_len + 4n + out_len) E
  composed                                    (in_len + 11n + 2 out_len) E: pad copy, four-step forward 4n (or 2n for a
                                              tuned n), multiply 3n, backward as forward, slice
Prints one JSON object per case (ms per step, GB/s of each arm's model where it has one, the ratios) and the card's name, power
limit and SM clock (nvidia-smi, read-only query) before and after."""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)

GiB = 1 << 30
# name, precision ("d" / "f"), n, (in_len, out_len); in_len = out_len = n / 2 unless given
CASES = [
    ("f32-4096", "f", 4096, None), ("f32-8192", "f", 8192, None), ("f32-2^16", "f", 1 << 16, None),
    ("f32-2^18", "f", 1 << 18, None), ("f32-2^20", "f", 1 << 20, None),
    ("f64-2048", "d", 2048, None), ("f64-8192", "d", 8192, None), ("f64-2^16", "d", 1 << 16, None),
    ("f64-2^20", "d", 1 << 20, None),
    ("f32-2^16-unpadded", "f", 1 << 16, (1 << 16, 1 << 16)),
]


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim, clk = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_clock": clk}
    except Exception as exc:   # the numbers still stand; the record says why the card state is missing
        return {"error": str(exc)}


def timed(torch, stream, fn, seconds, warmup):
    """ms per call of fn on `stream` (a torch stream), after warm-up, over enough calls to fill about `seconds`"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        for _ in range(warmup):
            fn()
        a.record(stream); fn(); b.record(stream)
        b.synchronize()
        steps = max(3, min(5000, int(seconds * 1e3 / max(a.elapsed_time(b), 1e-3))))
        a.record(stream)
        for _ in range(steps):
            fn()
        b.record(stream)
        b.synchronize()
    return a.elapsed_time(b) / steps, steps


def rel_l2(x, y):
    return float(((x - y).abs().double() ** 2).sum().sqrt() / (y.abs().double() ** 2).sum().sqrt())


def run_case(torch, dfft, name, prec, n, lens, seconds, warmup):
    li, lo = lens if lens else (n // 2, n // 2)
    P = dfft.DOUBLE if prec == "d" else dfft.FLOAT
    E = 16 if prec == "d" else 8
    cdt = torch.complex128 if prec == "d" else torch.complex64
    nlines = max(1, GiB // (li * E))
    g = torch.Generator(device="cuda")
    g.manual_seed(n)
    a = torch.randn(nlines, li, dtype=cdt, device="cuda", generator=g)
    m = torch.exp(2j * math.pi * torch.rand(n, dtype=torch.float64, device="cuda", generator=g)).to(cdt) / n
    out = torch.empty(nlines, lo, dtype=cdt, device="cuda")
    plan = dfft.LinesConvolvePlan(one_d=(n, nlines), padded=(li, lo), precision=P)
    lines = dfft.LinesPlan(n, 1, nlines, nlines, n, 0, precision=P)
    long_path = dfft.length_kind(n, P) != 2
    ps = torch.cuda.ExternalStream(plan.stream)
    ls = torch.cuda.ExternalStream(lines.stream)
    held = {}
    torch.cuda.synchronize()

    def run_plan():
        plan.execute(a.data_ptr(), out.data_ptr(), m.data_ptr(), 1)

    def run_composed():
        x = torch.nn.functional.pad(a, (0, n - li))
        lines.execute(x.data_ptr(), dfft.FORWARD)
        x.mul_(m)
        lines.execute(x.data_ptr(), dfft.BACKWARD)
        held["composed"] = x[:, :lo].contiguous()

    def run_torch():
        held["torch"] = torch.fft.ifft(torch.fft.fft(a, n=n) * m)[..., :lo]

    try:
        with torch.cuda.stream(ps):
            run_plan()
        with torch.cuda.stream(ls):
            run_composed()
        run_torch()
        torch.cuda.synchronize()
        err = {"composed": rel_l2(out, held["composed"]), "torch": rel_l2(out, held["torch"] * n)}
        res = {}
        for arm, st, fn in (("plan", ps, run_plan), ("composed", ls, run_composed), ("torch", torch.cuda.current_stream(), run_torch)):
            res[arm] = timed(torch, st, fn, seconds, warmup)
        torch.cuda.synchronize()
    finally:
        plan.destroy()
        lines.destroy()
    M = n * E
    fwd = 4 * n if long_path else 2 * n
    model = {"plan": ((li + (4 * n if long_path else 0) + lo) * E * nlines + M),
             "composed": ((li + n) + fwd + 3 * n + fwd + 2 * lo) * E * nlines + M}
    rec = {"case": name, "n": n, "in_len": li, "out_len": lo, "nlines": nlines, "path": "long" if long_path else "short",
           "ms": {k: round(v[0], 4) for k, v in res.items()}, "steps": {k: v[1] for k, v in res.items()},
           "model_GB": {k: round(v / 1e9, 3) for k, v in model.items()},
           "GBps": {k: round(model[k] / (res[k][0] * 1e-3) / 1e9, 1) for k in model},
           "plan_over_composed": round(res["plan"][0] / res["composed"][0], 3),
           "plan_over_torch": round(res["plan"][0] / res["torch"][0], 3),
           "rel_l2_vs": {k: float("%.3g" % v) for k, v in err.items()}}
    del a, out, m, held
    torch.cuda.empty_cache()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--case", action="append")
    args = ap.parse_args()
    import torch
    import distributedfft_b200 as dfft
    if not torch.cuda.is_available():
        sys.exit("conv_padded_bench needs a GPU")
    torch.cuda.set_device(0)
    print(json.dumps({"gpu_before": gpu_state(), "device": torch.cuda.get_device_name(0)}), flush=True)
    rows = []
    for name, prec, n, lens in CASES:
        if args.case and name not in args.case:
            continue
        rec = run_case(torch, dfft, name, prec, n, lens, args.seconds, args.warmup)
        rows.append(rec)
        print(json.dumps(rec), flush=True)
    print(json.dumps({"gpu_after": gpu_state()}), flush=True)
    print("%-20s %5s %6s %9s %9s %9s %8s %8s %8s" % ("case", "path", "nlines", "plan ms", "comp ms", "torch ms", "plan GB/s", "p/comp", "p/torch"))
    for r in rows:
        print("%-20s %5s %6d %9.3f %9.3f %9.3f %8.0f %8.3f %8.3f" % (r["case"], r["path"], r["nlines"], r["ms"]["plan"], r["ms"]["composed"],
                                                                  r["ms"]["torch"], r["GBps"]["plan"], r["plan_over_composed"],
                                                                  r["plan_over_torch"]))


if __name__ == "__main__":
    main()
