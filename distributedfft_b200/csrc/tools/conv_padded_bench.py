#!/usr/bin/env python
"""Zero-padded batched 1-D convolution, out[l] = ifft(fft(in[l], n) * m)[:out_len]: the padded convolve lines plan against the
sequence it replaces and against torch, one GPU (developer tool).

    python distributedfft_b200/csrc/tools/conv_padded_bench.py [--seconds 1.0] [--warmup 5] [--case NAME] [--real]

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
limit and SM clock (nvidia-smi, read-only query) before and after.

--real: the real plan, out[l] = irfft(rfft(in[l], n) * m, n)[:out_len] of real lines (one shared multiplier of n/2 + 1 points),
against these arms on the same seeded real lines (nlines chosen so that the real input holds about 1 GiB):
  plan      LinesConvolvePlan(one_d=(n, nlines), real_padded=(in_len, out_len)), out of place
  complex   the complex padded plan on the same lines widened to complex (widened once, untimed) with the Hermitian multiplier
  torch     torch.fft.irfft(torch.fft.rfft(a, n=n) * m, n=n)[..., :out_len] (cuFFT; the slice is a view)
Byte model, in complex elements E per line (two real lines per complex transform; M = n/2 + 1 points, or n for the complex plan):
  real plan, short path                       (in_len + out_len) / 2 E
  real plan, long path                        ((in_len + out_len) / 2 + 2n) E
  complex plan                                as above (in_len + out_len, or in_len + 4n + out_len)"""
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


REAL_CASES = ["f32-4096", "f32-8192", "f64-8192", "f32-2^16", "f64-2^16", "f32-2^18", "f32-2^20", "f64-2^20"]


def run_real_case(torch, dfft, name, prec, n, lens, seconds, warmup):
    li, lo = lens if lens else (n // 2, n // 2)
    P = dfft.DOUBLE if prec == "d" else dfft.FLOAT
    E = 16 if prec == "d" else 8
    rdt, cdt = (torch.float64, torch.complex128) if prec == "d" else (torch.float32, torch.complex64)
    nlines = max(1, GiB // (li * E // 2))
    g = torch.Generator(device="cuda")
    g.manual_seed(n)
    a = torch.randn(nlines, li, dtype=rdt, device="cuda", generator=g)
    H = n // 2 + 1
    m = torch.exp(2j * math.pi * torch.rand(H, dtype=torch.float64, device="cuda", generator=g)).to(cdt) / n
    m.imag[0] = 0                      # the complex arm's Hermitian multiplier has real bins 0 and n/2, as the C2R takes them
    if n % 2 == 0:
        m.imag[H - 1] = 0
    mfull = torch.cat([m, torch.conj(m[1: n - H + 1].flip(0))])
    aw = a.to(cdt)
    out = torch.empty(nlines, lo, dtype=rdt, device="cuda")
    outc = torch.empty(nlines, lo, dtype=cdt, device="cuda")
    plan = dfft.LinesConvolvePlan(one_d=(n, nlines), real_padded=(li, lo), precision=P)
    cplan = dfft.LinesConvolvePlan(one_d=(n, nlines), padded=(li, lo), precision=P)
    long_path = dfft.length_kind(n, P) != 2
    ps = torch.cuda.ExternalStream(plan.stream)
    cs = torch.cuda.ExternalStream(cplan.stream)
    held = {}
    torch.cuda.synchronize()

    def run_plan():
        plan.execute(a.data_ptr(), out.data_ptr(), m.data_ptr(), 1)

    def run_complex():
        cplan.execute(aw.data_ptr(), outc.data_ptr(), mfull.data_ptr(), 1)

    def run_torch():
        held["torch"] = torch.fft.irfft(torch.fft.rfft(a, n=n) * m, n=n)[..., :lo]

    try:
        with torch.cuda.stream(ps):
            run_plan()
        with torch.cuda.stream(cs):
            run_complex()
        run_torch()
        torch.cuda.synchronize()
        err = {"complex": rel_l2(out, outc.real), "torch": rel_l2(out, held["torch"] * n)}
        res = {}
        for arm, st, fn in (("plan", ps, run_plan), ("complex", cs, run_complex), ("torch", torch.cuda.current_stream(), run_torch)):
            res[arm] = timed(torch, st, fn, seconds, warmup)
        torch.cuda.synchronize()
    finally:
        plan.destroy()
        cplan.destroy()
    model = {"plan": ((li + lo) / 2 + (2 * n if long_path else 0)) * E * nlines + H * E,
             "complex": (li + lo + (4 * n if long_path else 0)) * E * nlines + n * E}
    rec = {"case": name, "real": True, "n": n, "in_len": li, "out_len": lo, "nlines": nlines, "path": "long" if long_path else "short",
           "ms": {k: round(v[0], 4) for k, v in res.items()}, "steps": {k: v[1] for k, v in res.items()},
           "model_GB": {k: round(v / 1e9, 3) for k, v in model.items()},
           "GBps": {k: round(model[k] / (res[k][0] * 1e-3) / 1e9, 1) for k in model},
           "plan_over_complex": round(res["plan"][0] / res["complex"][0], 3),
           "plan_over_torch": round(res["plan"][0] / res["torch"][0], 3),
           "rel_l2_vs": {k: float("%.3g" % v) for k, v in err.items()}}
    del a, aw, out, outc, m, mfull, held
    torch.cuda.empty_cache()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--case", action="append")
    ap.add_argument("--real", action="store_true", help="the real plan against the complex plan and torch (see above)")
    args = ap.parse_args()
    import torch
    import distributedfft_b200 as dfft
    if not torch.cuda.is_available():
        sys.exit("conv_padded_bench needs a GPU")
    torch.cuda.set_device(0)
    print(json.dumps({"gpu_before": gpu_state(), "device": torch.cuda.get_device_name(0)}), flush=True)
    rows = []
    for name, prec, n, lens in CASES:
        if args.case and name not in args.case or args.real and name not in REAL_CASES:
            continue
        rec = (run_real_case if args.real else run_case)(torch, dfft, name, prec, n, lens, args.seconds, args.warmup)
        rows.append(rec)
        print(json.dumps(rec), flush=True)
    print(json.dumps({"gpu_after": gpu_state()}), flush=True)
    if args.real:
        print("%-20s %5s %6s %9s %9s %9s %8s %8s %8s" % ("case", "path", "nlines", "plan ms", "cplx ms", "torch ms", "plan GB/s", "p/cplx",
                                                       "p/torch"))
        for r in rows:
            print("%-20s %5s %6d %9.3f %9.3f %9.3f %8.0f %8.3f %8.3f" % (r["case"], r["path"], r["nlines"], r["ms"]["plan"], r["ms"]["complex"],
                                                                      r["ms"]["torch"], r["GBps"]["plan"], r["plan_over_complex"],
                                                                      r["plan_over_torch"]))
        return
    print("%-20s %5s %6s %9s %9s %9s %8s %8s %8s" % ("case", "path", "nlines", "plan ms", "comp ms", "torch ms", "plan GB/s", "p/comp", "p/torch"))
    for r in rows:
        print("%-20s %5s %6d %9.3f %9.3f %9.3f %8.0f %8.3f %8.3f" % (r["case"], r["path"], r["nlines"], r["ms"]["plan"], r["ms"]["composed"],
                                                                  r["ms"]["torch"], r["GBps"]["plan"], r["plan_over_composed"],
                                                                  r["plan_over_torch"]))


if __name__ == "__main__":
    main()
