"""CPU tests of the batched 1-D convolve lines plans (dfft_lines_plan_create_convolve_1d / _r2c_1d) without a GPU.

dfft_debug_lines_conv_1d_ops records the one pass an execute launches, "LINE_CONV" or "LINE_CONV_R2C".  run_line_conv below gives
it its meaning -- "for every tile and line of the tile: numpy's FFT of the line, the product with the line's multiplier, the
inverse, unnormalised, the optional scale; stored through the output map" (for the real record: rfft, product, irfft with numpy's
C2R convention, the two lines of a pair `pair` elements apart) -- and the result is compared with ifft(fft(a) * m) * n and
irfft(rfft(a) * m, n) * n.  Every tuned length in both precisions, a multiplier shared by every line and one per line, scaled and
unscaled, in place and out of place, partial last tiles and odd line counts for R2C.  Every buffer starts NaN-filled with
canaries past its end, so a read outside a buffer, a missed store or a write past an end shows up; `in` (when distinct) and the
multiplier must come back unchanged.  The kernels' arithmetic is checked on the GPU by test_gpu_lines_conv1d.py."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_dry_run import IN, OUT
from test_lines_conv_dry_run import MULT, ConvMachine, check, code, rand_c
from test_r2c_dry_run import real_view
from test_real_lines_dry_run import CANARY, bufid


def run_line_conv(m, op):
    """LINE_CONV / LINE_CONV_R2C: tile t, line c (real: pair c, line h of the pair) at base + t*SB + c*cs (+ h*pair) + e*es on
    each side; the line's multiplier at mult + line * (0 if shared else n or n/2+1)"""
    real = op["op"] == "LINE_CONV_R2C"
    N, C, W = op["N"], op["C"], op["W"]
    _, SBi, csi, esi = op["ia"]
    _, SBo, cso, eso = op["oa"]
    ldi, ldo = op["pair"] if real else (0, 0)
    M = op["nzh"] if real else N
    assert not real or M == N // 2 + 1
    src, soff = real_view(m, op["in"], real)
    dst, doff = real_view(m, op["out"], real)
    mul, moff = m.view(op["mult"])
    e, j = np.arange(N), np.arange(M)
    staged = []
    for tile in range(op["ntiles"]):
        for c in range(C):
            for h in range(2 if real else 1):
                line = 2 * (tile * C + c) + h if real else tile * C + c
                if line >= W:
                    continue
                v = src[soff + tile * SBi + c * csi + h * ldi + e * esi]
                mk = mul[moff + (0 if op["shared"] else line * M) + j]
                if real:
                    x = np.fft.irfft(np.fft.rfft(v) * mk, n=N) * N
                else:
                    x = np.fft.ifft(np.fft.fft(v) * mk) * N
                if op["do_scale"]:
                    x = x * op["scale"]
                staged.append((tile, c, h, x))
    for tile, c, h, x in staged:
        dst[doff + tile * SBo + c * cso + h * ldo + e * eso] = x


def ops_of(n, nlines, real=False, flags=0, mult_count=1, precision=dfft.DOUBLE):
    return dfft.lines_conv_1d_ops(n, nlines, precision, real, flags, mult_count)


def simulate(n, nlines, a, M, real=False, flags=0, inplace=False, precision=dfft.DOUBLE):
    """a: [nlines][n] input; M: the multiplier, one line's (shared) or [nlines] of them"""
    H = n // 2 + 1
    mline = H if real else n
    mult_count = 1 if M.ndim == 1 else nlines
    io = -(-n * nlines // 2) if real else n * nlines   # complex128 slots holding the caller's buffer
    sizes = {IN: io, OUT: io, MULT: mline * mult_count}
    m = ConvMachine(sizes, inplace)
    inb = m.mem[IN].view(np.float64) if real else m.mem[IN]
    inb[: a.size] = a.reshape(-1)
    m.mem[MULT][: M.size] = M.reshape(-1)
    keep_in, keep_mult = m.mem[IN].copy(), m.mem[MULT].copy()
    ops = ops_of(n, nlines, real, flags, mult_count, precision)
    assert len(ops) == 1 and ops[0]["op"] == ("LINE_CONV_R2C" if real else "LINE_CONV")
    op = ops[0]
    assert (bufid(op["in"]), bufid(op["out"]), bufid(op["mult"])) == (IN, OUT, MULT)
    run_line_conv(m, op)
    assert np.array_equal(m.mem[MULT], keep_mult, equal_nan=True), "the multiplier was written"
    if not inplace:
        assert np.array_equal(m.mem[IN], keep_in, equal_nan=True), "`in` was written"
    for b, arr in m.mem.items():
        assert np.all(arr[sizes[b]:] == CANARY), f"write past the end of buffer {b}"
    out = m.mem[OUT].view(np.float64)[: n * nlines] if real else m.mem[OUT][: n * nlines]
    got = out.copy()
    assert not np.isnan(got.view(np.float64)).any(), "an output element was never written (or read NaN)"
    return got, op


def want_c2c(a, M, scaled):
    r = np.fft.ifft(np.fft.fft(a, axis=-1) * M, axis=-1)
    return r if scaled else r * a.shape[-1]


def want_r2c(a, M, scaled):
    n = a.shape[-1]
    r = np.fft.irfft(np.fft.rfft(a, axis=-1) * M, n=n, axis=-1)
    return r if scaled else r * n


PRECISIONS = [dfft.DOUBLE, dfft.FLOAT]


def tuned(precision):
    return sorted(dfft.supported_lengths(precision))


def test_every_tuned_length_has_both_kernels():
    for prec in PRECISIONS:
        lengths = tuned(prec)
        assert len(lengths) >= 26
        for n in lengths:
            assert dfft.length_kind(n, prec) == 2
            assert ops_of(n, 3, precision=prec)[0]["op"] == "LINE_CONV"
            assert ops_of(n, 3, real=True, precision=prec)[0]["op"] == "LINE_CONV_R2C"


@pytest.mark.parametrize("precision", PRECISIONS)
def test_c2c_convolution_matches_numpy_at_every_tuned_length(precision):
    for n in tuned(precision):
        C = ops_of(n, 1, precision=precision)[0]["C"]
        nlines = C + 1 if C > 1 else 3            # a partial last tile (for C == 1 every tile is whole)
        rng = np.random.default_rng(n * 7 + precision)
        a = rand_c(rng, (nlines, n))
        M = rand_c(rng, n)
        got, op = simulate(n, nlines, a, M, precision=precision)
        assert op["N"] == n and op["W"] == nlines and op["G"] == op["ntiles"] == -(-nlines // C)
        assert op["ia"] == op["oa"] == [0, C * n, n, 1] and op["inv"] == 0
        assert op["shared"] == 1 and not op["do_scale"]
        check(got, want_c2c(a, M, False))
        Mb = rand_c(rng, (nlines, n))
        got, op = simulate(n, nlines, a, Mb, flags=dfft.SCALE_BACKWARD, inplace=True, precision=precision)
        assert op["shared"] == 0 and op["do_scale"] and op["scale"] == pytest.approx(1.0 / n, rel=1e-15)
        check(got, want_c2c(a, Mb, True))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_r2c_convolution_matches_numpy_at_every_tuned_length(precision):
    for n in tuned(precision):
        C = ops_of(n, 1, real=True, precision=precision)[0]["C"]
        nlines = 2 * C + 1                         # odd: the last pair has no second line, and a partial last tile
        H = n // 2 + 1
        rng = np.random.default_rng(n * 11 + precision)
        a = rng.standard_normal((nlines, n))
        M = rand_c(rng, H)                         # not Hermitian: the C2R ignores what numpy's irfft ignores
        got, op = simulate(n, nlines, a, M, real=True, precision=precision)
        assert op["N"] == n and op["W"] == nlines and op["G"] == op["ntiles"] == -(-(-(-nlines // 2)) // C)
        assert op["ia"] == op["oa"] == [0, 2 * C * n, 2 * n, 1] and op["pair"] == [n, n] and op["nzh"] == H
        assert op["shared"] == 1 and not op["do_scale"]
        check(got, want_r2c(a, M, False))
        Mb = rand_c(rng, (nlines, H))
        for inplace in (False, True):
            got, op = simulate(n, nlines, a, Mb, real=True, flags=dfft.SCALE_BACKWARD, inplace=inplace, precision=precision)
            assert op["shared"] == 0 and op["do_scale"] and op["scale"] == pytest.approx(1.0 / n, rel=1e-15)
            check(got, want_r2c(a, Mb, True))


@pytest.mark.parametrize("real", [False, True])
def test_small_and_empty_batches(real):
    rng = np.random.default_rng(5)
    for n, nlines in ((16, 1), (1000, 2), (4, 1), (243, 5)):
        a = rng.standard_normal((nlines, n)) if real else rand_c(rng, (nlines, n))
        M = rand_c(rng, n // 2 + 1 if real else n)
        got, _ = simulate(n, nlines, a, M, real=real)
        check(got, (want_r2c if real else want_c2c)(a, M, False))
    op = ops_of(64, 0, real)[0]
    assert op["ntiles"] == 0 and op["W"] == 0
    # mult_count == nlines == 1 is the shared case
    assert ops_of(64, 1, real, mult_count=1)[0]["shared"] == 1


@pytest.mark.parametrize("real", [False, True])
def test_unsupported_requests_are_refused(real, monkeypatch):
    def c(n, nlines, flags=0, mult_count=1, precision=dfft.DOUBLE):
        return code(ops_of, n, nlines, real, flags, mult_count, precision)
    assert c(16, 4) == 0 and c(1000, 3) == 0 and c(16, 0) == 0 and c(16, 4, mult_count=4) == 0
    assert c(16, 4, flags=dfft.SCALE_BACKWARD) == 0
    for n in (7, 14, 22):                                    # generic lengths: no tuned kernel
        assert dfft.length_kind(n, dfft.DOUBLE) == 1
        assert c(n, 1) == -3 and c(n, 1, precision=dfft.FLOAT) == -3, n
    assert c(8192, 1) == -3                                  # beyond one shared-memory line (the four-step plan)
    assert c(17, 1) == -3                                    # no kernel at all
    if real:
        assert c(1, 4) == -3                                 # a real convolution needs n >= 2
    else:
        assert c(1, 4) == -3                                 # no C2C line of length 1
    assert c(0, 1) == -1 and c(-4, 1) == -1
    assert c(16, -1) == -1
    assert c(16, 1 << 31) == -3 and c(16, (1 << 31) - 1) == 0 and c(16, 1 << 62) == -3   # 2^31 lines
    assert c(16, 1, precision=7) == -1
    for flags in (dfft.DRY_RUN, dfft.NO_FUSE, dfft.NATURAL_SPECTRUM, dfft.SCALE_BACKWARD | 1, 1 << 31):
        assert c(16, 2, flags=flags) == -1, flags
    for mc in (0, 2, 5, -1):
        assert c(16, 4, mult_count=mc) == -1, mc
    assert c(512, 1) == 0
    monkeypatch.setenv("DFFT_VARIANT", "5")                  # an alternate tuning of 512: no line-convolution kernel
    assert c(512, 1) == -3
    monkeypatch.delenv("DFFT_VARIANT")
    monkeypatch.setenv("DFFT_GENERIC", "1")                  # run-time-scheduled entries have no line-convolution kernel
    assert c(16, 1) == -3
