"""Zero-padded 1-D convolve lines plans (LinesConvolvePlan(one_d=..., padded=(in_len, out_len)):
dfft_lines_plan_create_convolve_padded_1d) on the GPU.

out[l] = ifft(fft(in[l], n) * m)[:out_len] per line.  The reference is a long-double convolution per line (tests/ldfft.py) of the
precision-rounded input and multiplier; above 2^16 points every line is also held to scipy's fp64 FFT (ld_harness.ratios64) and
a few lines to long double.  Two transforms: the bounds of test_gpu_lines_conv1d.py with Ntot = n (twice the one-transform bounds).
Cases:
- short path (one kernel): every tuned length in both precisions with (in_len, out_len) = (n, n), (n/2, n/2 + 1), (1, n) and
  (n, 1), shared and per-line multipliers, scaled and unscaled, partial last tiles; bitwise equal to the circular plan
  (dfft_lines_plan_create_convolve_1d) at (n, n);
- long path (three passes, four-step): fp64 at 6144 (64 x 96), 8192, 2^16, 786432 and 10^6, fp32 at 8192, 2^18, 2^20 and 2^24,
  each split asserted from the plan's records, with (n/2, n/2), (n2 - 1, n - 1) and (n, n);
- more tiles than a 132-SM H100 holds resident CTAs in every pass, on both paths;
- bitwise: a shared multiplier against nlines identical copies, in place against out of place, three executes equal;
- fp32 at an odd complex64 offset; `in` and the multiplier unchanged and canaries intact around every buffer;
- agreement with the composed sequence: torch pad, LinesPlan forward, torch multiply, LinesPlan backward, slice;
- fp32 with a temporary past 2^31 elements (skipped, saying so, when free memory is short): sampled lines around element 2^31
  bitwise equal to a small plan over the same lines.
Each checked case prints a "CONVPAD-RATIO" line."""
import faulthandler
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from ld_harness import ratios64  # noqa: E402
from test_gpu_lines3d import CDT, EPS, PN, fenced  # noqa: E402
from test_gpu_lines_conv1d import run as run_circular  # noqa: E402
from test_gpu_lines_limits import LIMIT, free_or_skip, release  # noqa: E402

DOUBLE, FLOAT = dfft.DOUBLE, dfft.FLOAT
K_L2, K_LINF = 2 * ldfft.REL_L2_K, 2 * ldfft.LINF_K


@pytest.fixture(autouse=True)
def _watchdog(monkeypatch):
    faulthandler.dump_traceback_later(900, exit=True, file=sys.stderr)
    for var in ("DFFT_GENERIC", "DFFT_VARIANT"):
        monkeypatch.delenv(var, raising=False)
    yield
    faulthandler.cancel_dump_traceback_later()


def inputs(n, li, nlines, prec, per_line, seed):
    """(a[nlines][li], m): m is [n] or [nlines][n]; |m| in [0.5, 2), random phase"""
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((nlines, li)) + 1j * rng.standard_normal((nlines, li))
    mshape = ((nlines,) if per_line else ()) + (n,)
    m = rng.uniform(0.5, 2.0, mshape) * np.exp(2j * np.pi * rng.uniform(size=mshape))
    return a.astype(CDT[prec][0]), m.astype(CDT[prec][0])


def run(n, li, lo, nlines, prec, a, m, flags=0, inplace=False, offset=0, repeat=1):
    """one plan on fenced buffers, executed `repeat` times from the same input; returns the output [nlines][lo] as numpy"""
    torch.cuda.set_device(0)
    assert not inplace or li == lo
    plan = dfft.LinesConvolvePlan(one_d=(n, nlines), padded=(li, lo), precision=prec, flags=flags)
    tdt = CDT[prec][1]
    flat, mflat = np.ascontiguousarray(a).reshape(-1), np.ascontiguousarray(m).reshape(-1)
    mc = nlines if m.ndim == 2 else 1
    a_m, mult, mfence = fenced(mflat, tdt, offset)
    try:
        first = None
        for _ in range(repeat):
            a_in, inp, ifence = fenced(flat, tdt, offset)
            if inplace:
                a_out, out, ofence = a_in, inp, ifence
            else:
                a_out, out, ofence = fenced(nlines * lo, tdt, offset)
            torch.cuda.synchronize()                 # the plan runs on its own stream
            plan.execute(inp.data_ptr(), out.data_ptr(), mult.data_ptr(), mc)
            plan.synchronize()
            cur = out.cpu().numpy().copy()
            for arena, view, (lo_f, hi_f) in ((a_out, out, ofence), (a_m, mult, mfence)) + (() if inplace else ((a_in, inp, ifence),)):
                k = lo_f.numel()
                assert torch.equal(arena[:k], lo_f) and torch.equal(arena[k + view.numel():], hi_f), "canary overwritten"
            if not inplace:
                assert torch.equal(inp.cpu(), torch.from_numpy(flat)), "input changed"
            assert torch.equal(mult.cpu(), torch.from_numpy(mflat)), "multiplier changed"
            if first is None:
                first = cur
            else:
                assert same(cur, first), "executes differ"
            del a_in, inp, a_out, out
    finally:
        plan.destroy()
    assert not np.isnan(first.view(first.real.dtype)).any(), "unwritten output"
    return first.reshape(nlines, lo)


def ld_pad(a, m, n, lo, scaled=False):
    """long-double ifft(fft(zero_pad(a, n)) * m)[:, :lo] * n"""
    x = np.zeros((a.shape[0], n), dtype=np.clongdouble)
    x[:, : a.shape[1]] = a
    out = ldfft.fft(ldfft.fft(x, 1) * m.astype(np.clongdouble), 1, +1)[:, :lo]
    return out / n if scaled else out


def scipy_pad(a, m, n, lo, scaled=False):
    import scipy.fft
    y = scipy.fft.ifft(scipy.fft.fft(a.astype(np.complex128), n=n, axis=1, workers=-1) * m.astype(np.complex128), axis=1,
                       norm="backward" if scaled else "forward", workers=-1)
    return y[:, :lo]


def check(got, ref, prec, n, what, big=False):
    r = ratios64(got, ref, EPS[prec], max(n, 2)) if big else ldfft.ratios(got, ref, EPS[prec], max(n, 2))
    print(f"CONVPAD-RATIO {what} rel_l2 {r[0]:.3f} linf {r[1]:.3f}")
    assert r[0] <= K_L2 and r[1] <= K_LINF, (what, r)


def check_all(got, a, m, n, lo, prec, what, scaled=False):
    """long double for every line up to 2^16 points; beyond, scipy fp64 for every line and long double for the last (to 2^20)"""
    if n <= 1 << 16:
        check(got, ld_pad(a, m, n, lo, scaled), prec, n, what)
        return
    check(got, scipy_pad(a, m, n, lo, scaled), prec, n, what + ", scipy fp64", big=True)
    if n <= 1 << 20:
        ml = m[-1:] if m.ndim == 2 else m
        check(got[-1:], ld_pad(a[-1:], ml, n, lo, scaled), prec, n, what + ", last line long double")


def same(x, y):
    return x.shape == y.shape and np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8))


def ops(n, li, lo, nlines, prec):
    return dfft.lines_conv_padded_1d_ops(n, li, lo, nlines, prec)


def pad_cases(n):
    h = max(1, n // 2)
    return [(n, n), (h, min(n, h + 1)), (1, n), (n, 1)]


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_short_path_at_every_tuned_length(prec):
    lengths = sorted(dfft.supported_lengths(prec))
    assert len(lengths) >= 26, lengths
    for n in lengths:
        C = ops(n, n, n, 1, prec)[0]["C"]
        nlines = 3 * C + 1 + (C == 1)                # a partial last tile
        for i, (li, lo) in enumerate(pad_cases(n)):
            per_line, scaled = i % 2 == 1, i >= 2
            a, m = inputs(n, li, nlines, prec, per_line, seed=n * 13 + 5 * prec + i)
            got = run(n, li, lo, nlines, prec, a, m, flags=dfft.SCALE_BACKWARD if scaled else 0)
            check(got, ld_pad(a, m, n, lo, scaled), prec, n,
                  f"short n={n} ({li}, {lo}) x {nlines} {PN[prec]} {'per-line' if per_line else 'shared'}{' scaled' if scaled else ''}")
            if (li, lo) == (n, n):
                assert same(got, run_circular(n, nlines, prec, a, m, repeat=1)), ("padded (n, n) vs the circular plan", n)


# (n, precision, n1, n2, nlines)
LONG = [(6144, DOUBLE, 64, 96, 5), (8192, DOUBLE, 64, 128, 5), (1 << 16, DOUBLE, 256, 256, 3), (786432, DOUBLE, 768, 1024, 2),
        (10 ** 6, DOUBLE, 1000, 1000, 2), (8192, FLOAT, 64, 128, 5), (1 << 18, FLOAT, 512, 512, 3), (1 << 20, FLOAT, 1024, 1024, 2),
        (1 << 24, FLOAT, 4096, 4096, 2)]


@pytest.mark.parametrize("n,prec,n1,n2,nlines", LONG, ids=["%d%s" % (c[0], PN[c[1]]) for c in LONG])
def test_long_path(n, prec, n1, n2, nlines):
    assert dfft.length_kind(n, prec) != 2
    for i, (li, lo) in enumerate([(n // 2, n // 2), (n2 - 1, n - 1), (n, n)]):
        rec = ops(n, li, lo, nlines, prec)
        assert [o["op"] for o in rec] == ["XF_TW_PAD", "XCONV", "XB_TW_PAD"] and (rec[0]["N"], rec[1]["N"]) == (n1, n2), rec
        per_line, scaled = i % 2 == 0, i == 1
        a, m = inputs(n, li, nlines, prec, per_line, seed=n % 1000003 + i)
        got = run(n, li, lo, nlines, prec, a, m, flags=dfft.SCALE_BACKWARD if scaled else 0)
        check_all(got, a, m, n, lo, prec, f"long n={n} {n1}x{n2} ({li}, {lo}) x {nlines} {PN[prec]}"
                  f" {'per-line' if per_line else 'shared'}{' scaled' if scaled else ''}", scaled)


# more tiles in every pass than a 132-SM H100 holds resident CTAs (an SM holds at most 32 CTAs)
MANY = [(64, DOUBLE, 32, 33, 67601), (8192, DOUBLE, 4096, 4096, 1201), (4096, FLOAT, 2000, 3000, 4500), (10 ** 6, FLOAT, 300000, 500000, 20)]


@pytest.mark.parametrize("n,prec,li,lo,nlines", MANY)
def test_more_tiles_than_resident_ctas(n, prec, li, lo, nlines):
    for o in ops(n, li, lo, nlines, prec):
        assert o["ntiles"] > 132 * 32, (o["op"], o["ntiles"])
    a, m = inputs(n, li, nlines, prec, True, seed=n + prec)
    got = run(n, li, lo, nlines, prec, a, m)
    what = f"many n={n} ({li}, {lo}) x {nlines} {PN[prec]}"
    if n <= 64:
        check(got, ld_pad(a, m, n, lo), prec, n, what)
    else:   # every line against scipy's fp64 FFT, the last against long double
        check(got, scipy_pad(a, m, n, lo), prec, n, what + ", scipy fp64", big=True)
        check(got[-1:], ld_pad(a[-1:], m[-1], n, lo), prec, n, what + ", last line long double")


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_bitwise_identities(prec):
    """a shared multiplier vs nlines identical copies, in place vs out of place, three executes (run's repeat)"""
    for n, li, lo, nlines in ((64, 40, 40, 37), (1024, 512, 700, 9), (125, 125, 125, 11), (4096, 1, 4096, 5), (6144, 3000, 3000, 4),
                              (8192, 4096, 5000, 3), (36, 20, 30, 17), (1 << 16, 1 << 15, 1 << 15, 2)):
        a, m = inputs(n, li, nlines, prec, False, seed=n + 3)
        base = run(n, li, lo, nlines, prec, a, m, repeat=3)
        copies = np.ascontiguousarray(np.broadcast_to(m, (nlines, n)))
        assert same(base, run(n, li, lo, nlines, prec, a, copies)), ("copies", n)
        if li == lo:
            assert same(base, run(n, li, lo, nlines, prec, a, m, inplace=True)), ("in place", n)


def test_fp32_at_an_odd_complex64_offset():
    for n, li, lo, nlines in ((1024, 600, 1024, 5), (12, 5, 12, 130), (8192, 4096, 4097, 3), (36, 36, 1, 40)):
        for per_line in (False, True):
            a, m = inputs(n, li, nlines, FLOAT, per_line, seed=9 + n)
            got = run(n, li, lo, nlines, FLOAT, a, m, offset=1)
            check(got, ld_pad(a, m, n, lo), FLOAT, n, f"offset n={n} ({li}, {lo}) x {nlines} f32 {'per-line' if per_line else 'shared'}")


def composed(n, li, lo, nlines, prec, a, m):
    """the sequence the plan replaces: torch pad, LinesPlan forward, torch multiply, LinesPlan backward, slice"""
    x = torch.nn.functional.pad(torch.from_numpy(a).cuda(), (0, n - li)).contiguous()
    mt = torch.from_numpy(np.ascontiguousarray(m)).cuda()
    plan = dfft.LinesPlan(n, 1, nlines, nlines, n, 0, precision=prec)
    try:
        torch.cuda.synchronize()
        plan.execute(x.data_ptr(), dfft.FORWARD)
        plan.synchronize()
        x.mul_(mt)
        torch.cuda.synchronize()
        plan.execute(x.data_ptr(), dfft.BACKWARD)
        plan.synchronize()
    finally:
        plan.destroy()
    return x[:, :lo].cpu().numpy()


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_agrees_with_the_composed_sequence(prec):
    for n, li, lo, nlines in ((256, 100, 200, 37), (4096, 2048, 2049, 9), (1000, 1, 1000, 5), (8192, 4096, 4096, 7),
                              (6144, 3000, 6000, 3), (1 << 16, 1 << 15, 1 << 15, 3), (1 << 20, 1 << 19, 1 << 19, 2)):
        a, m = inputs(n, li, nlines, prec, True, seed=3 + n)
        got = run(n, li, lo, nlines, prec, a, m)
        check(got, composed(n, li, lo, nlines, prec, a, m), prec, n, f"vs composed n={n} ({li}, {lo}) x {nlines} {PN[prec]}")


def test_temporary_past_2_31_elements():
    """fp32 1024 x 1024 lines, 2049 of them: the temporary holds 2049 * 2^20 > 2^31 elements.  Lines 2047 and 2048 sit on either
    side of temporary element 2^31"""
    n, li, lo, nl = 1 << 20, 1 << 19, 1 << 19, 2049
    assert nl * n > LIMIT
    free_or_skip(nl * (n + li + lo) * 8, "padded convolve 2^20 x 2049 f32")
    rec = ops(n, li, lo, nl, FLOAT)
    assert [o["op"] for o in rec] == ["XF_TW_PAD", "XCONV", "XB_TW_PAD"] and rec[0]["N"] == 1024, rec
    idx = np.array([0, 1, 2046, 2047, 2048, nl - 1])
    rng = np.random.default_rng(8)
    m = (rng.uniform(0.5, 2.0, n) * np.exp(2j * np.pi * rng.uniform(size=n))).astype(np.complex64)
    g = torch.Generator(device="cuda")
    g.manual_seed(8)
    inp = torch.empty(nl * li, dtype=torch.complex64, device="cuda")
    for chunk in inp.split(1 << 28):
        torch.view_as_real(chunk).normal_(generator=g)
    out = torch.full((nl * lo,), float("nan"), dtype=torch.complex64, device="cuda")
    mult = torch.from_numpy(m).cuda()
    try:
        plan = dfft.LinesConvolvePlan(one_d=(n, nl), padded=(li, lo), precision=FLOAT)
        try:
            torch.cuda.synchronize()
            plan.execute(inp.data_ptr(), out.data_ptr(), mult.data_ptr(), 1)
            plan.synchronize()
        finally:
            plan.destroy()
        for chunk in out.split(1 << 27):
            assert not torch.isnan(torch.view_as_real(chunk)).any().item(), "unwritten output"
        x = inp.view(nl, li)[idx].cpu().numpy()
        got = out.view(nl, lo)[idx].cpu().numpy()
    finally:
        del inp, out
        release()
    small = run(n, li, lo, len(idx), FLOAT, x, m)
    assert same(got, small), "sampled lines against a small plan"
    check_all(got, x, m, n, lo, FLOAT, f"past 2^31 n={n} ({li}, {lo}) {len(idx)} sampled lines of {nl} f32")
