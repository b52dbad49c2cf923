#!/usr/bin/env python
"""Convolve plan against the three-call sequence it replaces, one GPU (developer tool).

    python distributedfft_b200/csrc/tools/conv_bench.py [--n 512] [--steps 20] [--rounds 3] [--float] [--real]

The sequence is what a user writes without the convolve plan: the default forward plan (transposed [y][z][x] spectrum), then
torch.mul(spectrum, m_transposed, out=<the backward plan's bufferDev1>), then the default backward plan.  The convolve plan gets the
same input and the multiplier in natural [x][y][z] order.  Both are created once; each round times `steps` iterations of one, then
the other, alternating, with CUDA events on the plans' stream, after untimed warm-up iterations.  Prints one JSON object: card
name, power limit and SM clock (nvidia-smi, read-only query) before and after, ms per convolution of every round, the error of the
convolve plan's output against the sequence's in units of eps * log2(Ntot) (the GPU tests' bound: 2.0 / 8.0), and the algorithmic
HBM bytes of each, from shapes, in units of one slab sweep E*M (E = elements, M = bytes per complex element)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "distributedfft_b200", "csrc", "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from r2c_bench import gpu_state  # noqa: E402


def algorithmic_bytes(n, h, esz, real, fwd_fused, bwd_fused):
    """HBM bytes of one convolution, from shapes: every pass reads and writes its array once (the fused t0 kernels keep their
    intermediate in L2), the multiply of the sequence reads two arrays and writes one, the fused X pass reads the spectrum and the
    multiplier and writes once.  Returns (sequence, convolve)."""
    S = n * n * h * esz                                          # the (half) spectrum
    if real:
        Rb = n ** 3 * esz // 2                                   # the real slab
        fwd_t0 = Rb + S + 2 * S                                  # real Z pass, Y pass in place
        bwd_t0 = 2 * S + S + Rb
    else:
        fwd_t0 = 2 * S if fwd_fused else 4 * S
        bwd_t0 = 2 * S if bwd_fused else 4 * S
    return fwd_t0 + 2 * S + 3 * S + 2 * S + bwd_t0, fwd_t0 + 3 * S + bwd_t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--float", action="store_true")
    ap.add_argument("--real", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    import distributedfft_b200 as dfft
    import ldfft

    n, real = args.n, args.real
    prec = dfft.FLOAT if args.float else dfft.DOUBLE
    rdt, cdt = (torch.float32, torch.complex64) if args.float else (torch.float64, torch.complex128)
    h = n // 2 + 1 if real else n
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randn(n ** 3, dtype=rdt if real else cdt, device="cuda", generator=gen)
    m = torch.randn(n * n * h, dtype=cdt, device="cuda", generator=gen)             # natural [x][y][z']
    out_conv = torch.empty_like(a)
    conv = dfft.fft_mpi_plan_dft_convolve_3d(n, n, n, a.data_ptr(), out_conv.data_ptr(), None, 0, 1, prec, 0, real=real)
    # the sequence: spectrum [y][z'][x] from the forward plan, multiplied into the backward plan's bufferDev1
    mt = m.reshape(n, n, h).permute(1, 2, 0).contiguous().reshape(-1)
    ncplx = n * n * h
    spec = torch.empty(ncplx, dtype=cdt, device="cuda")
    out_seq = torch.empty_like(a)
    if real:
        fwd = dfft.fft_mpi_plan_dft_r2c_3d(n, n, n, a.data_ptr(), spec.data_ptr(), None, 0, 1, dfft.FORWARD, prec)
        bwd = dfft.fft_mpi_plan_dft_r2c_3d(n, n, n, spec.data_ptr(), out_seq.data_ptr(), None, 0, 1, dfft.BACKWARD, prec)
    else:
        fwd = dfft.fft_mpi_plan_dft_c2c_3d(n, n, n, a.data_ptr(), spec.data_ptr(), None, 0, 1, dfft.FORWARD, prec)
        bwd = dfft.fft_mpi_plan_dft_c2c_3d(n, n, n, spec.data_ptr(), out_seq.data_ptr(), None, 0, 1, dfft.BACKWARD, prec)
    # a torch view of bwd's bufferDev1 (library-owned device memory), so the multiply writes it directly
    esz = spec.element_size()
    b1 = torch.as_tensor(_DevArray(bwd.bufferDev1, ncplx, "<c16" if not args.float else "<c8"), device="cuda")
    assert b1.data_ptr() == bwd.bufferDev1 and b1.numel() * esz == ncplx * esz
    st = torch.cuda.ExternalStream(conv.stream)
    assert fwd.stream and bwd.stream

    def run_conv():
        conv.execute_convolve(m.data_ptr())

    def run_seq():
        fwd.execute()
        ev = torch.cuda.ExternalStream(fwd.stream)
        with torch.cuda.stream(ev):
            torch.mul(spec, mt, out=b1)
        bwd_st = torch.cuda.ExternalStream(bwd.stream)
        bwd_st.wait_stream(ev)
        bwd.execute()
        st.wait_stream(bwd_st)

    def timed(fn, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ext = [torch.cuda.ExternalStream(p.stream) for p in (conv, fwd, bwd)]
        for s in ext[1:]:
            s.wait_stream(ext[0])
        e0.record(st)
        for _ in range(steps):
            for s in ext[1:]:
                s.wait_stream(st)
            fn()
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1) / steps

    state_before = gpu_state()
    for fn in (run_conv, run_seq):
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    rounds = []
    for _ in range(args.rounds):
        rounds.append({"conv_ms": timed(run_conv, args.steps), "seq_ms": timed(run_seq, args.steps)})
    torch.cuda.synchronize()
    got = out_conv.double() if real else out_conv.to(torch.complex128)
    ref = out_seq.double() if real else out_seq.to(torch.complex128)
    d = (got - ref).abs()
    u = ldfft.EPS["float" if args.float else "double"] * np.log2(n ** 3)
    rms = ref.abs().pow(2).mean().sqrt().item()
    err = {"rel_l2": (d.pow(2).sum().sqrt() / ref.abs().pow(2).sum().sqrt()).item() / u, "linf": d.max().item() / rms / u}
    seq_b, conv_b = algorithmic_bytes(n, h, esz, real, fwd.fused, bwd.fused)
    res = {
        "shape": [n, n, n], "precision": "float" if args.float else "double", "real": real, "steps": args.steps, "rounds": rounds,
        "conv_ms_median": float(np.median([r["conv_ms"] for r in rounds])), "seq_ms_median": float(np.median([r["seq_ms"] for r in rounds])),
        "conv_t": conv.timings(), "conv_pass_ms": conv.pass_timings(), "fwd_t": fwd.timings(), "bwd_t": bwd.timings(),
        "fwd_fused": fwd.fused, "bwd_fused": bwd.fused, "error_vs_sequence": err,
        "bytes_sequence": seq_b, "bytes_convolve": conv_b, "sweeps_sequence": seq_b / (n ** 3 * esz), "sweeps_convolve": conv_b / (n ** 3 * esz),
        "gpu_before": state_before, "gpu_after": gpu_state(),
    }
    for p in (conv, fwd, bwd):
        p.destroy()
    print(json.dumps(res))


class _DevArray:
    """__cuda_array_interface__ over a raw device pointer"""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}


if __name__ == "__main__":
    main()
