"""Real zero-padded 1-D convolve lines plans (LinesConvolvePlan(one_d=..., real_padded=(in_len, out_len)):
dfft_lines_plan_create_convolve_padded_r2c_1d) on the GPU.

out[l] = irfft(rfft(in[l], n) * m, n)[:out_len] per real line.  The reference is test_gpu_lines_conv1d.py's long-double real
convolution (imaginary parts of bins 0 and n/2 dropped) of the zero-padded, precision-rounded line, sliced; above 2^16 points every
line is also held to scipy's fp64 FFT (ld_harness.ratios64) and the last line to long double.  Two transforms: the bounds of
test_gpu_lines_conv1d.py with Ntot = n.  Cases:
- short path (one kernel): every tuned length in both precisions with (in_len, out_len) = (n, n), (n/2, n/2 + 1), (1, n) and
  (n, 1), shared and per-line multipliers, scaled and unscaled, odd line counts (the last pair has one line), partial last tiles;
  bitwise equal to the circular R2C plan (dfft_lines_plan_create_convolve_r2c_1d) at (n, n);
- long path (three passes over line pairs, four-step): fp64 at 6144 (64 x 96), 8192, 2^16, 16000 (125 x 128, odd n1) and 10^6,
  fp32 at 8192, 2^18, 2^20 and 2^24, each split asserted from the plan's records;
- more tiles than a 132-SM H100 holds resident CTAs in every pass, on both paths;
- bitwise: a shared multiplier against nlines identical copies, in place against out of place, three executes equal, and the
  imaginary parts of m[0] and m[n/2] ignored;
- fp32 at an odd float offset; `in` and the multiplier unchanged and canaries intact around every buffer;
- agreement with the complex padded plan run on the same lines widened to complex (with the Hermitian multiplier);
- fp32 with a temporary past 2^31 elements (skipped, saying so, when free memory is short): sampled line pairs around temporary
  element 2^31 bitwise equal to a small plan over the same lines.
Each checked case prints a "CONVPADR2C-RATIO" line."""
import faulthandler
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from ld_harness import ratios64  # noqa: E402
from test_gpu_lines3d import CDT, EPS, PN, RDT, fenced  # noqa: E402
from test_gpu_lines_conv1d import ld_conv1  # noqa: E402
from test_gpu_lines_conv1d import run as run_circular  # noqa: E402
from test_gpu_lines_conv_padded import run as run_complex  # noqa: E402
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
    """(a[nlines][li] real, m): m is [n/2+1] or [nlines][n/2+1]; |m| in [0.5, 2), random phase, also at bins 0 and n/2"""
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((nlines, li))
    mshape = ((nlines,) if per_line else ()) + (n // 2 + 1,)
    m = rng.uniform(0.5, 2.0, mshape) * np.exp(2j * np.pi * rng.uniform(size=mshape))
    return a.astype(RDT[prec][0]), m.astype(CDT[prec][0])


def run(n, li, lo, nlines, prec, a, m, flags=0, inplace=False, offset=0, repeat=1):
    """one plan on fenced buffers, executed `repeat` times from the same input; returns the output [nlines][lo] as numpy"""
    torch.cuda.set_device(0)
    assert not inplace or li == lo
    plan = dfft.LinesConvolvePlan(one_d=(n, nlines), real_padded=(li, lo), precision=prec, flags=flags)
    tdt = RDT[prec][1]
    flat, mflat = np.ascontiguousarray(a).reshape(-1), np.ascontiguousarray(m).reshape(-1)
    mc = nlines if m.ndim == 2 else 1
    a_m, mult, mfence = fenced(mflat, CDT[prec][1], offset)
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
    assert not np.isnan(first).any(), "unwritten output"
    return first.reshape(nlines, lo)


def zero_pad(a, n):
    x = np.zeros((a.shape[0], n), dtype=a.dtype)
    x[:, : a.shape[1]] = a
    return x


def ld_pad(a, m, n, lo, scaled=False):
    """long-double irfft(rfft(zero_pad(a, n)) * m, n)[:, :lo] * n (C2R convention at bins 0 and n/2)"""
    return ld_conv1(zero_pad(a, n), m, True, scaled)[:, :lo]


def scipy_pad(a, m, n, lo, scaled=False):
    import scipy.fft
    s = scipy.fft.rfft(a.astype(np.float64), n=n, axis=1, workers=-1) * m.astype(np.complex128)
    return scipy.fft.irfft(s, n=n, axis=1, norm="backward" if scaled else "forward", workers=-1)[:, :lo]


def check(got, ref, prec, n, what, big=False):
    r = ratios64(got, ref, EPS[prec], max(n, 2)) if big else ldfft.ratios(got, ref, EPS[prec], max(n, 2))
    print(f"CONVPADR2C-RATIO {what} rel_l2 {r[0]:.3f} linf {r[1]:.3f}")
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
    return dfft.lines_conv_padded_1d_ops(n, li, lo, nlines, prec, real=True)


def pad_cases(n):
    h = max(1, n // 2)
    return [(n, n), (h, min(n, h + 1)), (1, n), (n, 1)]


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_short_path_at_every_tuned_length(prec):
    lengths = sorted(dfft.supported_lengths(prec))
    assert len(lengths) >= 26, lengths
    for n in lengths:
        C = ops(n, n, n, 1, prec)[0]["C"]
        nlines = 2 * (2 * C + 1) + 1                 # odd: the last pair has one line; a partial last tile
        for i, (li, lo) in enumerate(pad_cases(n)):
            per_line, scaled = i % 2 == 1, i >= 2
            a, m = inputs(n, li, nlines, prec, per_line, seed=n * 13 + 5 * prec + i)
            got = run(n, li, lo, nlines, prec, a, m, flags=dfft.SCALE_BACKWARD if scaled else 0)
            check(got, ld_pad(a, m, n, lo, scaled), prec, n,
                  f"short n={n} ({li}, {lo}) x {nlines} {PN[prec]} {'per-line' if per_line else 'shared'}{' scaled' if scaled else ''}")
            if (li, lo) == (n, n):
                assert same(got, run_circular(n, nlines, prec, a, m, real=True, repeat=1)), ("real padded (n, n) vs the circular plan", n)


# (n, precision, n1, n2, nlines)
LONG = [(6144, DOUBLE, 64, 96, 5), (8192, DOUBLE, 64, 128, 5), (1 << 16, DOUBLE, 256, 256, 3), (16000, DOUBLE, 125, 128, 5),
        (10 ** 6, DOUBLE, 1000, 1000, 3), (8192, FLOAT, 64, 128, 5), (1 << 18, FLOAT, 512, 512, 3), (1 << 20, FLOAT, 1024, 1024, 3),
        (1 << 24, FLOAT, 4096, 4096, 3)]


@pytest.mark.parametrize("n,prec,n1,n2,nlines", LONG, ids=["%d%s" % (c[0], PN[c[1]]) for c in LONG])
def test_long_path(n, prec, n1, n2, nlines):
    assert dfft.length_kind(n, prec) != 2
    for i, (li, lo) in enumerate([(n // 2, n // 2), (n2 - 1, n - 1), (n, n)]):
        rec = ops(n, li, lo, nlines, prec)
        assert [o["op"] for o in rec] == ["XF_TW_PAD_R2C", "XCONV_R2C", "XB_TW_PAD_C2R"] and (rec[0]["N"], rec[1]["N"]) == (n1, n2), rec
        per_line, scaled = i % 2 == 0, i == 1
        a, m = inputs(n, li, nlines, prec, per_line, seed=n % 1000003 + i)
        got = run(n, li, lo, nlines, prec, a, m, flags=dfft.SCALE_BACKWARD if scaled else 0)
        check_all(got, a, m, n, lo, prec, f"long n={n} {n1}x{n2} ({li}, {lo}) x {nlines} {PN[prec]}"
                  f" {'per-line' if per_line else 'shared'}{' scaled' if scaled else ''}", scaled)


# more tiles in every pass than a 132-SM H100 holds resident CTAs (an SM holds at most 32 CTAs)
MANY = [(64, DOUBLE, 32, 33, 135203), (8192, DOUBLE, 4096, 4096, 2401), (4096, FLOAT, 2000, 3000, 8449), (10 ** 6, FLOAT, 300000, 500000, 39)]


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
    """a shared multiplier vs nlines identical copies, in place vs out of place, three executes (run's repeat), and the imaginary
    parts of m[0] and m[n/2] ignored"""
    for n, li, lo, nlines in ((64, 40, 40, 37), (1024, 512, 700, 9), (125, 125, 125, 11), (4096, 1, 4096, 5), (6144, 3000, 3000, 4),
                              (8192, 4096, 5000, 3), (36, 20, 30, 17), (2401, 1200, 1200, 5), (1 << 16, 1 << 15, 1 << 15, 3)):
        a, m = inputs(n, li, nlines, prec, False, seed=n + 3)
        base = run(n, li, lo, nlines, prec, a, m, repeat=3)
        copies = np.ascontiguousarray(np.broadcast_to(m, (nlines, n // 2 + 1)))
        assert same(base, run(n, li, lo, nlines, prec, a, copies)), ("copies", n)
        if li == lo:
            assert same(base, run(n, li, lo, nlines, prec, a, m, inplace=True)), ("in place", n)
        m2 = m.copy()
        m2[0] = m2[0].real + 1.5j
        if n % 2 == 0:
            m2[n // 2] = m2[n // 2].real - 0.75j
        assert same(base, run(n, li, lo, nlines, prec, a, m2)), ("imaginary parts of the edge bins", n)


def test_fp32_at_an_odd_float_offset():
    for n, li, lo, nlines in ((1024, 600, 1024, 5), (12, 5, 12, 131), (8192, 4096, 4097, 3), (36, 36, 1, 41)):
        for per_line in (False, True):
            a, m = inputs(n, li, nlines, FLOAT, per_line, seed=9 + n)
            got = run(n, li, lo, nlines, FLOAT, a, m, offset=1)
            check(got, ld_pad(a, m, n, lo), FLOAT, n, f"offset n={n} ({li}, {lo}) x {nlines} f32 {'per-line' if per_line else 'shared'}")


def hermitian(m, n):
    """the full [n] spectrum of a real filter whose half spectrum is m (imaginary parts of bins 0 and n/2 dropped)"""
    h = m.astype(np.complex128).copy()
    h[..., 0] = h[..., 0].real
    if n % 2 == 0:
        h[..., n // 2] = h[..., n // 2].real
    full = np.empty(m.shape[:-1] + (n,), dtype=np.complex128)
    full[..., : n // 2 + 1] = h
    full[..., n // 2 + 1:] = np.conj(h[..., 1: n - n // 2][..., ::-1])
    return full.astype(m.dtype)


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_agrees_with_the_complex_padded_plan_on_widened_lines(prec):
    for n, li, lo, nlines in ((256, 100, 200, 37), (4096, 2048, 2049, 9), (1000, 1, 1000, 5), (8192, 4096, 4096, 7),
                              (6144, 3000, 6000, 3), (1 << 16, 1 << 15, 1 << 15, 3), (1 << 20, 1 << 19, 1 << 19, 3)):
        a, m = inputs(n, li, nlines, prec, True, seed=3 + n)
        got = run(n, li, lo, nlines, prec, a, m)
        wide = run_complex(n, li, lo, nlines, prec, a.astype(CDT[prec][0]), hermitian(m, n))
        check(got, wide.real.astype(np.float64), prec, n, f"vs complex plan n={n} ({li}, {lo}) x {nlines} {PN[prec]}", big=True)


def test_temporary_past_2_31_elements():
    """fp32 1024 x 1024 lines, 4097 of them: the temporary holds 2049 line pairs of 2^20 points, past 2^31 elements.  Pairs 2046 and
    2047 sit below temporary element 2^31 and the last line (alone in pair 2048) above it"""
    n, li, lo, nl = 1 << 20, 1 << 19, 1 << 19, 4097
    assert (nl + 1) // 2 * n > LIMIT
    free_or_skip(nl * (li + lo) * 4 + (nl + 1) // 2 * n * 8, "real padded convolve 2^20 x 4097 f32")
    rec = ops(n, li, lo, nl, FLOAT)
    assert [o["op"] for o in rec] == ["XF_TW_PAD_R2C", "XCONV_R2C", "XB_TW_PAD_C2R"] and rec[0]["N"] == 1024, rec
    idx = np.array([0, 1, 4092, 4093, 4094, 4095, nl - 1])   # whole pairs, in the same pairing as the small plan's
    rng = np.random.default_rng(8)
    m = (rng.uniform(0.5, 2.0, n // 2 + 1) * np.exp(2j * np.pi * rng.uniform(size=n // 2 + 1))).astype(np.complex64)
    g = torch.Generator(device="cuda")
    g.manual_seed(8)
    inp = torch.empty(nl * li, dtype=torch.float32, device="cuda")
    for chunk in inp.split(1 << 28):
        chunk.normal_(generator=g)
    out = torch.full((nl * lo,), float("nan"), dtype=torch.float32, device="cuda")
    mult = torch.from_numpy(m).cuda()
    try:
        plan = dfft.LinesConvolvePlan(one_d=(n, nl), real_padded=(li, lo), precision=FLOAT)
        try:
            torch.cuda.synchronize()
            plan.execute(inp.data_ptr(), out.data_ptr(), mult.data_ptr(), 1)
            plan.synchronize()
        finally:
            plan.destroy()
        for chunk in out.split(1 << 28):
            assert not torch.isnan(chunk).any().item(), "unwritten output"
        x = inp.view(nl, li)[idx].cpu().numpy()
        got = out.view(nl, lo)[idx].cpu().numpy()
    finally:
        del inp, out
        release()
    small = run(n, li, lo, len(idx), FLOAT, x, m)
    assert same(got, small), "sampled lines against a small plan"
    check_all(got, x, m, n, lo, FLOAT, f"past 2^31 n={n} ({li}, {lo}) {len(idx)} sampled lines of {nl} f32")
