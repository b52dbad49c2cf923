"""Batched 1-D convolve lines plans (LinesConvolvePlan(one_d=...): dfft_lines_plan_create_convolve_1d / _r2c_1d) on the GPU.

The reference is a long-double convolution per line (tests/ldfft.py; the real one with test_gpu_r2c.py's Hermitian extension,
imaginary parts of bins 0 and n/2 dropped) of the precision-rounded input and multiplier.  There are two transforms, so the
bounds are test_gpu_lines_conv.py's with Ntot = n: rel_l2 <= 2 * eps * log2(n) and max error / rms(ref) <= 8 * eps * log2(n).
Cases:
- every tuned length in both precisions, both kernels (fft_line_conv_kernel, fft_line_conv_r2c_kernel), shared and per-line
  multipliers, scaled and unscaled, with line counts that leave the last tile partial (R2C: odd, so the last pair has one line);
  R2C multipliers have nonzero imaginary parts at bins 0 and n/2;
- more tiles than a 132-SM H100 holds resident CTAs, at a few lengths;
- bitwise: a shared multiplier against nlines identical copies; in place against out of place; three executes equal; R2C with
  odd nlines against nlines + 1 lines whose last line (and its multiplier) is zero, on the first nlines lines;
- agreement with the three calls the plan replaces (LinesPlan / RealLinesPlan forward, torch multiply, backward);
- fp32 at an odd complex64 offset;
- `in` and the multiplier unchanged, canaries around every buffer.
Each case prints a "LINESCONV1D-RATIO" line."""
import faulthandler
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from test_gpu_lines3d import CDT, EPS, PN, RDT, fenced  # noqa: E402

DOUBLE, FLOAT = dfft.DOUBLE, dfft.FLOAT
K_L2, K_LINF = 2 * ldfft.REL_L2_K, 2 * ldfft.LINF_K


@pytest.fixture(autouse=True)
def _watchdog(monkeypatch):
    faulthandler.dump_traceback_later(900, exit=True, file=sys.stderr)
    for var in ("DFFT_GENERIC", "DFFT_VARIANT"):
        monkeypatch.delenv(var, raising=False)
    yield
    faulthandler.cancel_dump_traceback_later()


def inputs(n, nlines, prec, real, per_line, seed):
    """(a[nlines][n], m): m is one line's multiplier, or [nlines] of them; |m| in [0.5, 2), random phase (real: also at bins 0
    and n/2, whose imaginary parts the C2R ignores)"""
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((nlines, n))
    if not real:
        a = a + 1j * rng.standard_normal(a.shape)
    mshape = ((nlines,) if per_line else ()) + (n // 2 + 1 if real else n,)
    m = rng.uniform(0.5, 2.0, mshape) * np.exp(2j * np.pi * rng.uniform(size=mshape))
    return a.astype(RDT[prec][0] if real else CDT[prec][0]), m.astype(CDT[prec][0])


def run(n, nlines, prec, a, m, real=False, flags=0, inplace=False, offset=0, repeat=3):
    """one plan on fenced buffers, executed `repeat` times from the same input; returns the output as numpy"""
    torch.cuda.set_device(0)
    plan = dfft.LinesConvolvePlan(one_d=(n, nlines), precision=prec, real=real, flags=flags)
    tdt = RDT[prec][1] if real else CDT[prec][1]
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
                a_out, out, ofence = fenced(flat.size, tdt, offset)
            torch.cuda.synchronize()                 # the plan runs on its own stream
            plan.execute(inp.data_ptr(), out.data_ptr(), mult.data_ptr(), mc)
            plan.synchronize()
            cur = out.cpu().numpy().copy()
            for arena, view, (lo, hi) in ((a_out, out, ofence), (a_m, mult, mfence)) + (() if inplace else ((a_in, inp, ifence),)):
                k = lo.numel()
                assert torch.equal(arena[:k], lo) and torch.equal(arena[k + view.numel():], hi), "canary overwritten"
            if not inplace:
                assert torch.equal(inp.cpu(), torch.from_numpy(flat)), "input changed"
            assert torch.equal(mult.cpu(), torch.from_numpy(mflat)), "multiplier changed"
            if first is None:
                first = cur
            else:
                assert np.array_equal(cur.view(np.uint8), first.view(np.uint8)), "executes differ"
    finally:
        plan.destroy()
    assert not np.isnan(first.view(RDT[prec][0])).any(), "unwritten output"
    return first.reshape(a.shape)


def ld_conv1(a, m, real, scaled=False):
    """long-double ifft(fft(a) * m) * n (real: irfft(rfft(a) * m, n) * n) per line"""
    n = a.shape[1]
    s = ldfft.fft(a.astype(np.clongdouble), 1)
    ml = m.astype(np.clongdouble)
    if real:
        H = n // 2 + 1
        y = s[:, :H] * ml
        y[:, 0] = y[:, 0].real                        # what a C2R ignores: imaginary parts of bins 0 and n/2
        if n % 2 == 0:
            y[:, H - 1] = y[:, H - 1].real
        full = np.empty(a.shape, dtype=np.clongdouble)
        full[:, :H] = y
        full[:, H:] = np.conj(y[:, 1: n - H + 1][:, ::-1])
        out = ldfft.fft(full, 1, +1).real
    else:
        out = ldfft.fft(s * ml, 1, +1)
    return out / n if scaled else out


def check(got, ref, prec, what):
    rl2, linf = ldfft.ratios(got, ref, EPS[prec], max(got.shape[1], 2))
    print(f"LINESCONV1D-RATIO {what} rel_l2 {rl2:.3f} linf {linf:.3f}")
    assert rl2 <= K_L2 and linf <= K_LINF, (what, rl2, linf)


def same(x, y):
    return np.array_equal(x.view(np.uint8), y.view(np.uint8))


def tile_C(n, prec, real):
    return dfft.lines_conv_1d_ops(n, 1, prec, real)[0]["C"]


def tuned(prec):
    return sorted(dfft.supported_lengths(prec))


@pytest.mark.parametrize("real", [False, True])
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_every_tuned_length(prec, real):
    lengths = tuned(prec)
    assert len(lengths) >= 26, lengths
    kind = "r2c" if real else "c2c"
    for n in lengths:
        C = tile_C(n, prec, real)
        nlines = 2 * (3 * C) + 1 if real else 3 * C + 1 + (C == 1)   # partial last tile; R2C: odd
        for per_line in (False, True):
            a, m = inputs(n, nlines, prec, real, per_line, seed=n * 13 + 5 * prec + per_line + 2 * real)
            ref = ld_conv1(a, m, real)
            for scaled in (False, True):
                got = run(n, nlines, prec, a, m, real=real, flags=dfft.SCALE_BACKWARD if scaled else 0, repeat=3 if scaled else 1)
                check(got, ref / n if scaled else ref, prec,
                      f"{kind} n={n} x {nlines} {PN[prec]} {'per-line' if per_line else 'shared'}{' scaled' if scaled else ''}")


# more tiles than resident CTAs: a 132-SM H100 holds at most 2048 / (threads per CTA) CTAs per SM (fewer where registers or
# shared memory run out), so every line count below gives more tiles than 132 * 2048 / (T * C); partial last tiles throughout.
# (n, precision, real, nlines): T * C = 128 threads at 64 fp64, 1024 fp64, 4 fp32 and 768 fp32, 256 at 4096 fp64, 200 at 1000 fp32
MANY = [(64, DOUBLE, False, 65539), (1024, DOUBLE, True, 6001), (4096, DOUBLE, False, 601), (1000, FLOAT, False, 4197),
        (768, FLOAT, False, 5003), (4, FLOAT, True, (1 << 20) + 1)]


@pytest.mark.parametrize("n,prec,real,nlines", MANY)
def test_more_tiles_than_resident_ctas(n, prec, real, nlines):
    C = tile_C(n, prec, real)
    tiles = -(-(-(-nlines // 2) if real else nlines) // C)
    assert tiles > 132 * 16 or (n, tiles) in ((4096, 601), (1000, 2099)), (n, tiles)
    a, m = inputs(n, nlines, prec, real, True, seed=n + prec)
    got = run(n, nlines, prec, a, m, real=real, repeat=1)
    check(got, ld_conv1(a, m, real), prec, f"many {'r2c' if real else 'c2c'} n={n} x {nlines} {PN[prec]}")


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_bitwise_identities(prec):
    """a shared multiplier vs nlines identical copies, in place vs out of place, odd R2C vs a zero extra line"""
    for n, real in ((4, False), (64, False), (1024, False), (768, False), (4096, False), (125, False),
                    (16, True), (1024, True), (1000, True), (243, True), (4096, True)):
        C = tile_C(n, prec, real)
        nlines = 2 * (5 * C) + 1 if real else 5 * C + 3
        a, m = inputs(n, nlines, prec, real, False, seed=n + 3)
        base = run(n, nlines, prec, a, m, real=real, repeat=2)
        copies = np.ascontiguousarray(np.broadcast_to(m, (nlines,) + m.shape))
        assert same(base, run(n, nlines, prec, a, copies, real=real, repeat=1)), ("copies", n, real)
        assert same(base, run(n, nlines, prec, a, m, real=real, inplace=True, repeat=1)), ("in place", n, real)
        if real:
            # the missing second line of the last pair loads 0 and reads a 0 multiplier: the same bits as a zero line whose
            # own multiplier is zero
            _, mb = inputs(n, nlines, prec, real, True, seed=n + 4)
            odd = run(n, nlines, prec, a, mb, real=True, repeat=1)
            a1 = np.concatenate([a, np.zeros((1, n), a.dtype)])
            m1 = np.concatenate([mb, np.zeros((1,) + mb.shape[1:], mb.dtype)])
            even = run(n, nlines + 1, prec, a1, m1, real=True, repeat=1)
            assert same(odd, np.ascontiguousarray(even[:nlines])), ("odd vs zero line", n)


def three_calls(n, nlines, prec, a, m, real):
    """the sequence the plan replaces: forward lines plan, torch multiply, backward lines plan"""
    mt = torch.from_numpy(np.ascontiguousarray(m)).cuda()
    x = torch.from_numpy(a.reshape(-1).copy()).cuda()
    if real:
        plan = dfft.RealLinesPlan(n, nlines, precision=prec)
        s = torch.empty(nlines * (n // 2 + 1), dtype=CDT[prec][1], device="cuda")
        torch.cuda.synchronize()
        plan.execute(x.data_ptr(), s.data_ptr(), dfft.FORWARD)
        plan.synchronize()
        s.view(nlines, -1).mul_(mt)
        torch.cuda.synchronize()
        plan.execute(s.data_ptr(), x.data_ptr(), dfft.BACKWARD)
    else:
        plan = dfft.LinesPlan(n, 1, nlines, nlines, n, 0, precision=prec)
        torch.cuda.synchronize()
        plan.execute(x.data_ptr(), dfft.FORWARD)
        plan.synchronize()
        x.view(a.shape).mul_(mt)
        torch.cuda.synchronize()
        plan.execute(x.data_ptr(), dfft.BACKWARD)
    plan.synchronize()
    plan.destroy()
    return x.cpu().numpy().reshape(a.shape)


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_agrees_with_the_three_call_sequence(prec):
    for n, nlines, real in ((256, 37, False), (1024, 9, False), (1000, 5, False), (49, 11, False),
                            (1024, 9, True), (4096, 3, True), (9, 17, True), (768, 6, True)):
        a, m = inputs(n, nlines, prec, real, True, seed=3 + n)
        got = run(n, nlines, prec, a, m, real=real, repeat=1)
        torch.cuda.synchronize()
        check(got, three_calls(n, nlines, prec, a, m, real), prec, f"vs three calls {'r2c' if real else 'c2c'} n={n} x {nlines} {PN[prec]}")


def test_fp32_at_an_odd_complex64_offset():
    for n, nlines in ((1024, 5), (12, 130), (768, 3)):
        for per_line in (False, True):
            a, m = inputs(n, nlines, FLOAT, False, per_line, seed=9 + n)
            got = run(n, nlines, FLOAT, a, m, offset=1)
            check(got, ld_conv1(a, m, False), FLOAT, f"offset n={n} x {nlines} f32 {'per-line' if per_line else 'shared'}")
