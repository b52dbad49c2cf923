"""Real lines plans (RealLinesPlan: dfft_lines_plan_create_r2c / _r2c_2d, dfft_lines_execute_real) on the GPU.

Held to the bounds of the other long-double matrices (tests/ldfft.py, tests/ld_harness.py): rel_l2 <= 1.0 * eps * log2(n) and
max error / rms(ref) <= 4 * eps * log2(n), n = the real axis length for 1-D and nx * ny for 2-D.  Cases:
- every tuned length in both precisions on the tuned real kernels (fft_real.cuh), forward and C2R, odd and even line counts;
- the run-time-scheduled real kernels (fft_generic_r2c / c2r_kernel): lengths covering radices 2 .. 13, odd and single-stage
  lengths, the shared-memory limits 6400 fp64 / 12800 fp32, and every tuned length again under DFFT_GENERIC=1;
- far more tiles than resident CTAs; 2-D plans with odd and generic nx, generic ny, batches 1 and odd;
- fp32 complex data at an odd complex64 offset, and a refused misaligned fp64 complex buffer;
- the forward result against the first n/2+1 bins of a C2C LinesPlan on the same data widened to complex.
The backward input is not Hermitian (C2R ignores the imaginary parts at bin 0 and, even n, n/2).  Outputs are NaN-prefilled and
fenced with canaries, every plan executes three times with bitwise-equal results, and the input must be unchanged.  Worst ratios
per family are printed on "RLINES-RATIO" lines."""
import faulthandler
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from ld_harness import ratios64  # noqa: E402

DOUBLE, FLOAT = dfft.DOUBLE, dfft.FLOAT
FWD, BWD = dfft.FORWARD, dfft.BACKWARD
RDT = {DOUBLE: (np.float64, torch.float64), FLOAT: (np.float32, torch.float32)}
CDT = {DOUBLE: (np.complex128, torch.complex128), FLOAT: (np.complex64, torch.complex64)}
EPS = {DOUBLE: ldfft.EPS["double"], FLOAT: ldfft.EPS["float"]}
PN = {DOUBLE: "f64", FLOAT: "f32"}
CANARY = 64
WORST = {}


@pytest.fixture(autouse=True)
def _watchdog(monkeypatch):
    faulthandler.dump_traceback_later(240, exit=True, file=sys.stderr)
    for var in ("DFFT_GENERIC", "DFFT_VARIANT"):
        monkeypatch.delenv(var, raising=False)
    yield
    faulthandler.cancel_dump_traceback_later()


@pytest.fixture(scope="module", autouse=True)
def _long_double():
    assert np.finfo(np.longdouble).eps <= ldfft.LD_EPS_MAX, "np.longdouble is not wider than double: no reference for the fp64 bounds"


def fenced(host, tdt, offset=0):
    """device arena [canary | offset | data | canary]; `host` is flat numpy, or an int length for a NaN-filled output"""
    d = torch.device("cuda", 0)
    n = host if isinstance(host, int) else host.size
    rng = np.random.default_rng(99)
    pat = rng.standard_normal(2 * CANARY) if not tdt.is_complex else rng.standard_normal(2 * CANARY) + 1j * rng.standard_normal(2 * CANARY)
    pat = torch.from_numpy(pat).to(tdt).to(d)
    lo = CANARY + offset
    arena = torch.zeros(lo + n + CANARY, dtype=tdt, device=d)
    arena[:CANARY], arena[lo + n:] = pat[:CANARY], pat[CANARY:]
    if isinstance(host, int):
        arena[lo: lo + n] = float("nan")
    else:
        arena[lo: lo + n] = torch.from_numpy(host).to(d)
    return arena, arena[lo: lo + n], (arena[:lo].clone(), arena[lo + n:].clone())


def run(direction, dev_in, prec, n=None, nlines=0, two_d=None, offset=0, repeat=3):
    """one RealLinesPlan on fenced buffers, executed `repeat` times; `offset`: elements between the canary and the complex-side
    view; returns the output as numpy"""
    torch.cuda.set_device(0)
    nx, rows = (n, nlines) if two_d is None else (two_d[0], two_d[1] * two_d[2])
    rc, cc = rows * nx, rows * (nx // 2 + 1)
    fwd = direction == FWD
    in_t, out_t = (RDT[prec][1], CDT[prec][1]) if fwd else (CDT[prec][1], RDT[prec][1])
    n_in, n_out = (rc, cc) if fwd else (cc, rc)
    assert dev_in.size == n_in
    a_in, inp, _ = fenced(dev_in, in_t, 0 if fwd else offset)
    a_out, out, (lo, hi) = fenced(n_out, out_t, offset if fwd else 0)
    plan = dfft.RealLinesPlan(n, nlines, prec, two_d)
    try:
        first = None
        for _ in range(repeat):
            plan.execute(inp.data_ptr(), out.data_ptr(), direction)
            plan.synchronize()
            cur = out.cpu().numpy().copy()
            if first is None:
                first = cur
            else:
                assert np.array_equal(cur.view(np.uint8), first.view(np.uint8)), "executes differ"
    finally:
        plan.destroy()
    torch.cuda.synchronize()
    k = lo.numel()
    assert torch.equal(a_out[:k], lo) and torch.equal(a_out[k + n_out:], hi), "canary overwritten"
    assert torch.equal(inp.cpu(), torch.from_numpy(dev_in)), "input changed"
    assert not np.isnan(first.view(RDT[prec][0])).any(), "unwritten output"
    return first


# ---- long-double references ----------------------------------------------------------------------------------------------
def ld_rfft(x, axes):
    """x real (..., ny, nx) -> transform along `axes` (1-D: (-1,), 2-D: (-1, -2)), cut to nx//2+1 on the last axis"""
    y = x.astype(np.longdouble) + 0j
    for ax in axes:
        y = ldfft.fft(y, ax, -1)
    return y[..., : x.shape[-1] // 2 + 1]


def ld_irfft(S, nx, ny_axis=False):
    """numpy.fft.irfft(S, nx) * nx (with ny_axis: irfft2 * nx*ny, the inverse along axis -2 first), imaginary parts of bin 0 and
    (even nx) nx/2 dropped"""
    y = S.astype(np.clongdouble)
    if ny_axis:
        y = ldfft.fft(y, -2, +1)
    H = nx // 2 + 1
    y[..., 0] = y[..., 0].real
    if nx % 2 == 0:
        y[..., H - 1] = y[..., H - 1].real
    full = np.empty(y.shape[:-1] + (nx,), dtype=np.clongdouble)
    full[..., :H] = y
    full[..., H:] = np.conj(y[..., 1: nx - H + 1][..., ::-1])
    return ldfft.fft(full, -1, +1).real


def check(family, prec, got, ref, ntot, label, big=False):
    rl2, linf = (ratios64 if big else ldfft.ratios)(got.reshape(-1), np.asarray(ref).reshape(-1), EPS[prec], ntot)
    print("RLINES-RATIO %-10s %-44s rel_l2 %6.3f  linf %6.3f" % (family, label, rl2, linf))
    w = WORST.get((family, prec), (0.0, 0.0))
    WORST[family, prec] = (max(w[0], rl2), max(w[1], linf))
    assert rl2 <= ldfft.REL_L2_K and linf <= ldfft.LINF_K, (label, rl2, linf)


def one_d(family, n, nlines, prec, seed=0):
    rng = np.random.default_rng(n * 31 + nlines + seed)
    H = n // 2 + 1
    x = rng.standard_normal((nlines, n)).astype(RDT[prec][0])
    got = run(FWD, x.reshape(-1), prec, n, nlines)
    check(family, prec, got, ld_rfft(x, (-1,)), n, "fwd n=%d lines=%d %s" % (n, nlines, PN[prec]))
    S = (rng.standard_normal((nlines, H)) + 1j * rng.standard_normal((nlines, H))).astype(CDT[prec][0])
    got = run(BWD, S.reshape(-1), prec, n, nlines)
    check(family, prec, got, ld_irfft(S, n), n, "bwd n=%d lines=%d %s" % (n, nlines, PN[prec]))


def tuned(prec):
    return [n for n in dfft.supported_lengths(prec) if dfft.length_kind(n, prec) == 2]


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_every_tuned_length(prec):
    lengths = tuned(prec)
    assert len(lengths) >= 20, lengths
    for n in lengths:
        for nlines in (7, 8):
            one_d("tuned", n, nlines, prec)


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_forced_generic_kernel_on_tuned_lengths(prec, monkeypatch):
    lengths = tuned(prec)                       # before DFFT_GENERIC: under it no length reports a tuned kernel
    assert len(lengths) >= 20, lengths
    monkeypatch.setenv("DFFT_GENERIC", "1")     # read when a plan looks up its length
    assert all(dfft.length_kind(n, prec) == 1 for n in lengths)
    for n in lengths:
        one_d("forced-gen", n, 7, prec)


GENERIC_LENGTHS = [2, 3, 5, 7, 11, 13, 14, 21, 22, 26, 121, 169, 143, 360, 480, 1331, 2197, 1001, 3000]


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_generic_lengths(prec):
    limit = 6400 if prec == DOUBLE else 12800
    for n in GENERIC_LENGTHS + [limit]:
        assert dfft.length_kind(n, prec) == 1, n
        for nlines in ((1, 5) if n < 1000 else (3,)):
            one_d("generic", n, nlines, prec)
    with pytest.raises(dfft.DfftError, match=r"\(-3\)"):
        dfft.RealLinesPlan(2 * limit, 2, prec)


# far more tiles than resident CTAs: the grid-stride loop and the buffer reuse across tiles.  A CTA of these kernels has at least
# 128 threads (256 for the run-time-scheduled ones), so an SM holds at most 16 (8) of them; the line count gives every possible
# resident CTA three tiles, plus a lone last line.  Reference: long double for 14 points, scipy's fp64 FFT (ratios64: its own
# error is about 1 unit at these lengths) for the longer lines
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
@pytest.mark.parametrize("n,max_ctas,ref", [(512, 16, "scipy"), (360, 8, "scipy"), (14, 8, "ld")])
def test_many_tiles(prec, n, max_ctas, ref):
    import scipy.fft
    need = 3 * torch.cuda.get_device_properties(0).multi_processor_count * max_ctas
    nlines = 2 * dfft.real_lines_ops(n, 2, FWD, prec)[0]["C"] * need + 1
    assert dfft.real_lines_ops(n, nlines, FWD, prec)[0]["ntiles"] >= need
    rng = np.random.default_rng(n)
    H = n // 2 + 1
    x = rng.standard_normal((nlines, n)).astype(RDT[prec][0])
    S = (rng.standard_normal((nlines, H)) + 1j * rng.standard_normal((nlines, H))).astype(CDT[prec][0])
    if ref == "ld":
        want_f, want_b = ld_rfft(x, (-1,)), ld_irfft(S, n)
    else:
        want_f = scipy.fft.rfft(x.astype(np.float64), axis=1, workers=-1)
        want_b = scipy.fft.irfft(S.astype(np.complex128), n=n, axis=1, workers=-1) * n
    got = run(FWD, x.reshape(-1), prec, n, nlines, repeat=2)
    check("many-tiles", prec, got, want_f, n, "fwd n=%d lines=%d %s" % (n, nlines, PN[prec]), big=ref != "ld")
    got = run(BWD, S.reshape(-1), prec, n, nlines, repeat=2)
    check("many-tiles", prec, got, want_b, n, "bwd n=%d lines=%d %s" % (n, nlines, PN[prec]), big=ref != "ld")


# (nx, ny, batch): tuned, odd and generic nx; generic ny; batches 1 and odd
SHAPES_2D = [(1024, 64, 2), (64, 48, 3), (9, 16, 1), (125, 21, 3), (14, 12, 1), (360, 22, 3), (21, 26, 5)]


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
@pytest.mark.parametrize("nx,ny,batch", SHAPES_2D)
def test_2d(prec, nx, ny, batch):
    rng = np.random.default_rng(nx * 7 + ny + batch)
    H = nx // 2 + 1
    two_d = (nx, ny, batch)
    a = rng.standard_normal((batch, ny, nx)).astype(RDT[prec][0])
    got = run(FWD, a.reshape(-1), prec, two_d=two_d)
    check("2d", prec, got, ld_rfft(a, (-1, -2)), nx * ny, "fwd %dx%d batch %d %s" % (ny, nx, batch, PN[prec]))
    S = (rng.standard_normal((batch, ny, H)) + 1j * rng.standard_normal((batch, ny, H))).astype(CDT[prec][0])
    got = run(BWD, S.reshape(-1), prec, two_d=two_d)
    check("2d", prec, got, ld_irfft(S, nx, ny_axis=True), nx * ny, "bwd %dx%d batch %d %s" % (ny, nx, batch, PN[prec]))


@pytest.mark.parametrize("n", [768, 9, 360])
def test_fp32_complex_at_odd_complex64_offset(n):
    rng = np.random.default_rng(n)
    nlines, H = 5, n // 2 + 1
    x = rng.standard_normal((nlines, n)).astype(np.float32)
    got = run(FWD, x.reshape(-1), FLOAT, n, nlines, offset=1)
    check("offset", FLOAT, got, ld_rfft(x, (-1,)), n, "fwd n=%d complex64 offset 1" % n)
    S = (rng.standard_normal((nlines, H)) + 1j * rng.standard_normal((nlines, H))).astype(np.complex64)
    got = run(BWD, S.reshape(-1), FLOAT, n, nlines, offset=1)
    check("offset", FLOAT, got, ld_irfft(S, n), n, "bwd n=%d complex64 offset 1" % n)
    got = run(FWD, x.reshape(-1), FLOAT, two_d=(n, nlines, 1), offset=1)
    check("offset", FLOAT, got, ld_rfft(x[None], (-1, -2)), n * nlines, "2d fwd %dx%d complex64 offset 1" % (nlines, n))


def test_misaligned_fp64_complex_is_refused():
    r = torch.zeros(4 * 64, dtype=torch.float64, device="cuda")
    c = torch.zeros(4 * 33 + 1, dtype=torch.complex128, device="cuda")
    p = dfft.RealLinesPlan(64, 4)
    try:
        with pytest.raises(dfft.DfftError, match=r"\(-1\)"):
            p.execute(r.data_ptr(), c.data_ptr() + 8, FWD)
        with pytest.raises(dfft.DfftError, match=r"\(-1\)"):
            p.execute(c.data_ptr() + 8, r.data_ptr(), BWD)
        p.execute(r.data_ptr(), c.data_ptr(), FWD)
        p.synchronize()
    finally:
        p.destroy()


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
@pytest.mark.parametrize("n", [512, 1024, 125, 360, 13])
def test_forward_matches_c2c_lines_plan(prec, n):
    """the R2C half spectra equal the first n/2+1 bins of the C2C LinesPlan on the widened data"""
    nlines, H = 9, n // 2 + 1
    x = np.random.default_rng(n + 1).standard_normal((nlines, n)).astype(RDT[prec][0])
    got = run(FWD, x.reshape(-1), prec, n, nlines)
    z = torch.from_numpy(x.astype(CDT[prec][0])).to("cuda")
    lp = dfft.LinesPlan(n, 1, nlines, nlines, n, 0, prec)
    try:
        lp.execute(z.data_ptr(), FWD)
        lp.synchronize()
    finally:
        lp.destroy()
    c2c = z.cpu().numpy()[:, :H]
    check("vs-c2c", prec, got, c2c.astype(np.clongdouble), n, "n=%d %s" % (n, PN[prec]))


def test_zz_report_worst_ratios():
    for (family, prec), (rl2, linf) in sorted(WORST.items()):
        print("RLINES-RATIO worst %-10s %s rel_l2 %6.3f  linf %6.3f" % (family, PN[prec], rl2, linf))
