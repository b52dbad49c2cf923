#!/usr/bin/env python
"""Batched 3-D (or, with --dims 2 / --dims 1, 2-D / 1-D) spectral convolution: the convolve lines plan against the three calls it
replaces, one GPU (developer tool).

    python distributedfft_b200/csrc/tools/lines_conv_bench.py [--dims 3|2|1] [--steps 30] [--rounds 3] [--warmup 5] [--case NAME]

Every case convolves `batch` volumes (images, lines) with one multiplier of unit modulus / N (so repeated in-place steps keep
their magnitude).  The arms get the same seeded data:
  shared   LinesConvolvePlan, one multiplier for every volume (mult_count = 1), out of place
  pervol   the same plan with `batch` identical copies of the multiplier (mult_count = batch)
  noplane  (--dims 2, square 16 / 32 / 64 images) the plan created under DFFT_NO_PLANE=1 (X, XCONV, inverse X), shared
           multiplier; the shared and pervol plans are then created under DFFT_FORCE_PLANE=1, so that the one-kernel
           convolution is timed whatever kPlaneConvUse says
  3call    LinesPlan(three_d=... / two_d=... / n, nlines) forward in place, torch multiply by the shared multiplier, LinesPlan backward
           (real: RealLinesPlan forward into a spectrum buffer, multiply, backward into the output)
  torch    torch.fft.fftn * m -> ifftn over the last 3 / 2 / 1 axes (rfftn / irfftn for real cases; cuFFT, for context)
Before timing, the outputs of all arms are compared: shared against pervol and noplane with torch.equal (bit-identical by
construction), 3call and torch by rel_l2 against shared.  Each round times `steps` executes of each arm with CUDA events on the
arm's own stream (the plans' streams; torch's current stream for torch), arms alternating, after `warmup` untimed executes.

Prints one JSON object per case and a summary table: ms per step (median of the rounds), conv / 3call, and the HBM sweep model
of each arm in bytes with its GB/s at the measured time (V = one sweep of the batch, M = the multiplier as read):
  3-D C2C plane shape  conv 6V + M      3call 10V + M
  3-D C2C other        conv 10V + M     3call 14V + M
  3-D real             conv 2Vr + 8Vc + M   3call 2Vr + 12Vc + M   (Vr: real data, Vc: the half spectra)
  2-D C2C plane shape  conv 2V + M      noplane 6V + M    3call 10V + M
  2-D C2C other        conv 6V + M      3call 10V + M
  2-D real             conv 2Vr + 4Vc + M   3call 2Vr + 8Vc + M
  1-D C2C              conv 2V + M      3call 6V + M
  1-D real             conv 2Vr + M     3call 2Vr + 4Vc + M
Card name, power limit and SM clock (nvidia-smi, read-only query) are printed before and after."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)

# name, precision ("d" / "f"), (nx, ny, nz, batch), real.  128^3 has no plane kernel; 48^3 is a non-power-of-two plane
CASES = [
    ("16^3x16384", "d", (16, 16, 16, 16384), False), ("32^3x2048", "d", (32, 32, 32, 2048), False),
    ("64^3x256", "d", (64, 64, 64, 256), False), ("128^3x32", "d", (128, 128, 128, 32), False),
    ("48^3x512", "d", (48, 48, 48, 512), False),
    ("16^3x16384-f32", "f", (16, 16, 16, 16384), False), ("32^3x2048-f32", "f", (32, 32, 32, 2048), False),
    ("64^3x256-f32", "f", (64, 64, 64, 256), False),
    ("real-64^3x256", "d", (64, 64, 64, 256), True),
]
# --dims 2: (nx, ny, batch), about 2^26 complex elements per batch.  48^2 has no plane kernel
CASES_2D = [
    ("16^2x262144", "d", (16, 16, 262144), False), ("32^2x65536", "d", (32, 32, 65536), False),
    ("64^2x16384", "d", (64, 64, 16384), False),
    ("16^2x262144-f32", "f", (16, 16, 262144), False), ("32^2x65536-f32", "f", (32, 32, 65536), False),
    ("64^2x16384-f32", "f", (64, 64, 16384), False),
    ("48^2x16384", "d", (48, 48, 16384), False), ("256^2x1024", "d", (256, 256, 1024), False),
    ("1024^2x64", "d", (1024, 1024, 64), False),
    ("real-64^2x16384", "d", (64, 64, 16384), True), ("real-512^2x256", "d", (512, 512, 256), True),
]
# --dims 1: (n, nlines), about 2^26 complex elements per batch; 768 is mixed radix
CASES_1D = [
    ("256x262144", "d", (256, 262144), False), ("1024x65536", "d", (1024, 65536), False), ("4096x16384", "d", (4096, 16384), False),
    ("1024x65536-f32", "f", (1024, 65536), False), ("768x87381", "d", (768, 87381), False),
    ("real-1024x65536", "d", (1024, 65536), True), ("real-4096x16384", "d", (4096, 16384), True),
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


def make_conv(dfft, key, shape, prec, real, env):
    """LinesConvolvePlan with `env` (DFFT_NO_PLANE / DFFT_FORCE_PLANE) set at creation only"""
    if env:
        os.environ[env] = "1"
    try:
        return dfft.LinesConvolvePlan(**{key: shape}, precision=prec, real=real)
    finally:
        if env:
            os.environ.pop(env)


def run_case(torch, np, dfft, case, args):
    name, p, shape, real = case
    two, one = len(shape) == 3, len(shape) == 2
    nx, batch = shape[0], shape[-1]
    spatial = tuple(reversed(shape[:-1]))                                             # (nz, ny, nx), (ny, nx) or (n,)
    key = "one_d" if one else "two_d" if two else "three_d"
    prec = dfft.FLOAT if p == "f" else dfft.DOUBLE
    rdt, cdt = (torch.float32, torch.complex64) if p == "f" else (torch.float64, torch.complex128)
    er = 4 if p == "f" else 8
    ec = 2 * er
    H = nx // 2 + 1
    N = int(np.prod(spatial))
    mx = H if real else nx
    mshape = spatial[:-1] + (mx,)
    dims = tuple(range(-len(spatial), 0))
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn((batch,) + spatial, dtype=rdt if real else cdt, device="cuda", generator=gen)
    phase = torch.rand(mshape, dtype=rdt, device="cuda", generator=gen) * (2 * np.pi)
    m1 = (torch.polar(torch.ones_like(phase), phase) / N).to(cdt).contiguous()
    mb = m1.expand((batch,) + mshape).contiguous()
    plane_shape = two and not real and shape[0] == shape[1] and shape[0] in (16, 32, 64)
    conv = make_conv(dfft, key, shape, prec, real, "DFFT_FORCE_PLANE" if plane_shape else None)
    noplane = make_conv(dfft, key, shape, prec, real, "DFFT_NO_PLANE") if plane_shape else None
    if one:
        fwd = dfft.RealLinesPlan(nx, batch, precision=prec) if real else dfft.LinesPlan(nx, 1, batch, batch, nx, 0, precision=prec)
    else:
        fwd = dfft.RealLinesPlan(**{key: shape}, precision=prec) if real else dfft.LinesPlan(**{key: shape}, precision=prec)
    try:
        y = {k: torch.empty_like(x) for k in ("shared", "pervol") + (("noplane",) if noplane else ())}
        z = x.clone()                                                                 # the three-call arm's buffer
        spec = torch.empty((batch,) + spatial[:-1] + (H,), dtype=cdt, device="cuda") if real else None
        zout = torch.empty_like(x) if real else z

        def three_calls():
            if real:
                fwd.execute(x.data_ptr(), spec.data_ptr(), dfft.FORWARD)
                spec.mul_(m1)
                fwd.execute(spec.data_ptr(), zout.data_ptr(), dfft.BACKWARD)
            else:
                fwd.execute(z.data_ptr(), dfft.FORWARD)
                z.mul_(m1)
                fwd.execute(z.data_ptr(), dfft.BACKWARD)

        def torch_arm():
            if real:
                return torch.fft.irfftn(torch.fft.rfftn(x, dim=dims) * m1, s=spatial, dim=dims)
            return torch.fft.ifftn(torch.fft.fftn(x, dim=dims) * m1, dim=dims)

        jobs = {
            "shared": (conv.stream, lambda: conv.execute(x.data_ptr(), y["shared"].data_ptr(), m1.data_ptr(), 1)),
            "pervol": (conv.stream, lambda: conv.execute(x.data_ptr(), y["pervol"].data_ptr(), mb.data_ptr(), batch)),
        }
        if noplane:
            jobs["noplane"] = (noplane.stream, lambda: noplane.execute(x.data_ptr(), y["noplane"].data_ptr(), m1.data_ptr(), 1))
        jobs["3call"] = (fwd.stream, three_calls)
        jobs["torch"] = (None, torch_arm)
        # cross-check before timing: one step of every arm from the same input
        torch.cuda.synchronize()
        for k in y:
            jobs[k][1]()
        conv.synchronize()
        if noplane:
            noplane.synchronize()
        with torch.cuda.stream(torch.cuda.ExternalStream(fwd.stream)):
            three_calls()
        fwd.synchronize()
        t_out = torch_arm() * N                                                       # torch's ifftn is normalised
        torch.cuda.synchronize()
        ref = y["shared"]

        def rel(a):
            return float(torch.linalg.vector_norm(a - ref) / torch.linalg.vector_norm(ref))
        check = {"shared_eq_pervol": bool(torch.equal(y["shared"], y["pervol"])), "rel_l2_3call": rel(zout), "rel_l2_torch": rel(t_out)}
        if noplane:
            check["shared_eq_noplane"] = bool(torch.equal(y["shared"], y["noplane"]))
        del t_out
        for st, fn in jobs.values():
            with torch.cuda.stream(torch.cuda.ExternalStream(st) if st is not None else torch.cuda.current_stream()):
                for _ in range(args.warmup):
                    fn()
        torch.cuda.synchronize()
        rounds = []
        for _ in range(args.rounds):
            rounds.append({k: time_steps(torch, st, fn, args.steps) for k, (st, fn) in jobs.items()})
        torch.cuda.synchronize()
    finally:
        conv.destroy()
        fwd.destroy()
        if noplane:
            noplane.destroy()
    med = {k: float(np.median([r[k] for r in rounds])) for k in rounds[0]}
    if one:
        plane = False
    elif two:
        plane = plane_shape
    else:
        plane = dfft.lines_conv_3d_ops(*shape, prec, real)[0]["op"] == "XY_PLANE"
    Mimg = ec * N // nx * mx
    Msh, Mpv = Mimg, Mimg * batch
    if real:
        Vr, Vc = er * N * batch, ec * N // nx * H * batch
        if one:
            conv_b, call_b = 2 * Vr, 2 * Vr + 4 * Vc
            model = "conv 2Vr+M, 3call 2Vr+4Vc+M"
        else:
            conv_b, call_b = (2 * Vr + 4 * Vc, 2 * Vr + 8 * Vc) if two else (2 * Vr + 8 * Vc, 2 * Vr + 12 * Vc)
            model = "conv 2Vr+4Vc+M, 3call 2Vr+8Vc+M" if two else "conv 2Vr+8Vc+M, 3call 2Vr+12Vc+M"
    else:
        V = ec * N * batch
        if one:
            conv_b, call_b = 2 * V, 6 * V
            model = "conv 2V+M, 3call 6V+M"
        elif two:
            conv_b, call_b = (2 * V if plane else 6 * V), 10 * V
            model = "conv 2V+M, noplane 6V+M, 3call 10V+M" if plane else "conv 6V+M, 3call 10V+M"
        else:
            conv_b, call_b = (6 * V, 10 * V) if plane else (10 * V, 14 * V)
            model = "conv 6V+M, 3call 10V+M" if plane else "conv 10V+M, 3call 14V+M"
    model_bytes = {"shared": conv_b + Msh, "pervol": conv_b + Mpv, "3call": call_b + Msh}
    if noplane:
        model_bytes["noplane"] = 6 * V + Msh
    res = {
        "case": name, "precision": "float" if p == "f" else "double", "shape": list(shape), "real": real, "plane_kernel": plane,
        "steps": args.steps, "rounds": rounds, "median_ms": med,
        "ratio_shared_vs_3call": med["shared"] / med["3call"], "ratio_pervol_vs_3call": med["pervol"] / med["3call"],
        "ratio_shared_vs_noplane": med["shared"] / med["noplane"] if noplane else None,
        "sweep_model": model, "model_bytes": model_bytes,
        "model_gbps": {k: b / med[k] / 1e6 for k, b in model_bytes.items()}, "cross_check": check,
    }
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--case", action="append", help="run only these cases (default: all)")
    ap.add_argument("--dims", type=int, choices=(1, 2, 3), default=3, help="3-D volumes (default), 2-D images or 1-D lines")
    args = ap.parse_args()
    import numpy as np
    import torch
    import distributedfft_b200 as dfft

    torch.cuda.set_device(0)
    for var in ("DFFT_NO_PLANE", "DFFT_FORCE_PLANE", "DFFT_GENERIC", "DFFT_VARIANT"):
        os.environ.pop(var, None)
    print(json.dumps({"gpu_before": gpu_state()}), flush=True)
    results = []
    for case in {1: CASES_1D, 2: CASES_2D, 3: CASES}[args.dims]:
        if args.case and case[0] not in args.case:
            continue
        r = run_case(torch, np, dfft, case, args)
        results.append(r)
        print(json.dumps(r), flush=True)
    print(json.dumps({"gpu_after": gpu_state()}), flush=True)
    print("%-16s %5s %9s %9s %9s %9s %6s %6s %7s %7s %7s  %s" % (
        "case", "plane", "shared", "pervol", "3call", "torch", "sh/3c", "pv/3c", "GB/s_sh", "GB/s_pv", "GB/s_3c", "cross-check"))
    for r in results:
        m, g, c = r["median_ms"], r["model_gbps"], r["cross_check"]
        print("%-16s %5s %9.3f %9.3f %9.3f %9.3f %6.3f %6.3f %7.0f %7.0f %7.0f  eq=%s 3call=%.1e torch=%.1e" % (
            r["case"], "on" if r["plane_kernel"] else "off", m["shared"], m["pervol"], m["3call"], m["torch"],
            r["ratio_shared_vs_3call"], r["ratio_pervol_vs_3call"], g["shared"], g["pervol"], g["3call"],
            c["shared_eq_pervol"], c["rel_l2_3call"], c["rel_l2_torch"]))
        if "noplane" in m:
            print("%-16s noplane %9.3f ms  GB/s %7.0f  shared/noplane %6.3f  eq=%s" % (
                r["case"], m["noplane"], g["noplane"], r["ratio_shared_vs_noplane"], c["shared_eq_noplane"]))


if __name__ == "__main__":
    main()
