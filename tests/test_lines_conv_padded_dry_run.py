"""CPU tests of the zero-padded 1-D convolve lines plans (dfft_lines_plan_create_convolve_padded_1d) without a GPU.

dfft_debug_lines_conv_padded_1d_ops records the passes one execute launches: "LINE_CONV_PAD" (short path), or "XF_TW_PAD", "XCONV"
and "XB_TW_PAD" (long path, four-step).  The interpreters below give the new records their meaning and run_xconv (the 2-D and 3-D
convolve plans' column pass) the middle one; the result is compared with ifft(fft(a, n) * m)[:, :out_len] * n.  Every buffer starts
NaN-filled with canaries past its end, so a read past nlines * in_len, an output element left unwritten or a write past
nlines * out_len shows up; `in` (when distinct) and the multiplier must come back unchanged.  The kernels' arithmetic is checked on
the GPU by test_gpu_lines_conv_padded.py."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_dry_run import IN, OUT
from test_lines_conv_dry_run import MULT, TEMP, ConvMachine, code, rand_c, run_xconv
from test_real_lines_dry_run import CANARY, bufid

PRECISIONS = [dfft.DOUBLE, dfft.FLOAT]


def run_line_conv_pad(m, op):
    """LINE_CONV_PAD: line tile*C + c at base + tile*SB + c*cs + e*es on each side; points e < in_len are read, the rest are zero;
    FFT, the product with the line's multiplier, the inverse (unnormalised), the optional scale; points e < out_len are stored"""
    N, C, W = op["N"], op["C"], op["W"]
    _, SBi, csi, esi = op["ia"]
    _, SBo, cso, eso = op["oa"]
    li, lo = op["in_len"], op["out_len"]
    src, soff = m.view(op["in"])
    dst, doff = m.view(op["out"])
    mul, moff = m.view(op["mult"])
    ei, eo = np.arange(li), np.arange(lo)
    staged = []
    for tile in range(op["ntiles"]):
        for c in range(C):
            line = tile * C + c
            if line >= W:
                continue
            v = np.zeros(N, dtype=np.complex128)
            v[:li] = src[soff + tile * SBi + c * csi + ei * esi]
            x = np.fft.ifft(np.fft.fft(v) * mul[moff + (0 if op["shared"] else line * N) + np.arange(N)]) * N
            if op["do_scale"]:
                x = x * op["scale"]
            staged.append((tile, c, x))
    for tile, c, x in staged:   # every line is read before any is stored: in place is allowed when in_len == out_len
        dst[doff + tile * SBo + c * cso + eo * eso] = x[:lo]


def run_four_step_pad(m, op):
    """XF_TW_PAD: per line a (ia.SA apart) and column col = b*C + c < W: point e at offset b*SB + c*cs + e*es inside the line, read
    only where that offset is < in_len (zero otherwise); FFT; twiddle e^{-2 pi i col*k / tw_n}; stored through the output map.
    XB_TW_PAD: per line and row col: the row through the input map; twiddle e^{+2 pi i col*k / tw_n}; inverse FFT (unnormalised);
    point e stored where its offset b*SB + c*cs + e*es inside the output line (oa.SA apart) is < out_len"""
    fwd = op["op"] == "XF_TW_PAD"
    N, C, G, W, tw = op["N"], op["C"], op["G"], op["W"], op["tw_n"]
    SAi, SBi, csi, esi = op["ia"]
    SAo, SBo, cso, eso = op["oa"]
    assert op["tstore"] == (1 if fwd else 0) and op["inv"] == (0 if fwd else 1) and not op["do_scale"]
    src, soff = m.view(op["in"])
    dst, doff = m.view(op["out"])
    e = np.arange(N)
    staged = []
    for tile in range(op["ntiles"]):
        a, b = divmod(tile, G)
        for c in range(C):
            col = b * C + c
            if col >= W:
                continue
            rel = b * SBi + c * csi + e * esi
            v = np.zeros(N, dtype=np.complex128)
            ok = rel < op["in_len"] if fwd else np.ones(N, bool)
            v[ok] = src[soff + a * SAi + rel[ok]]
            w = np.exp(-2j * np.pi * ((col * e) % tw) / tw)
            x = np.fft.fft(v) * w if fwd else np.fft.ifft(v * np.conj(w)) * N
            staged.append((a, b, c, x))
    for a, b, c, x in staged:
        rel = b * SBo + c * cso + e * eso
        ok = np.ones(N, bool) if fwd else rel < op["out_len"]
        dst[doff + a * SAo + rel[ok]] = x[ok]


def ops_of(n, in_len, out_len, nlines, flags=0, mult_count=1, precision=dfft.DOUBLE):
    return dfft.lines_conv_padded_1d_ops(n, in_len, out_len, nlines, precision, flags, mult_count)


def simulate(n, in_len, out_len, nlines, a, M, flags=0, inplace=False, precision=dfft.DOUBLE):
    """a: [nlines][in_len] input; M: the multiplier, [n] (shared) or [nlines][n]"""
    mult_count = 1 if M.ndim == 1 else nlines
    sizes = {IN: nlines * in_len, OUT: nlines * out_len, MULT: n * mult_count, TEMP: nlines * n}
    m = ConvMachine(sizes, inplace)
    m.mem[IN][: a.size] = a.reshape(-1)
    m.mem[MULT][: M.size] = M.reshape(-1)
    keep_in, keep_mult = m.mem[IN].copy(), m.mem[MULT].copy()
    ops = ops_of(n, in_len, out_len, nlines, flags, mult_count, precision)
    for op in ops:
        assert bufid(op["out"]) != MULT and (inplace or bufid(op["out"]) != IN), ("a pass writes a read-only buffer", op["op"])
        assert op["op"] == "XCONV" or (op["in_len"], op["out_len"]) == (in_len, out_len)
        if op["op"] == "LINE_CONV_PAD":
            run_line_conv_pad(m, op)
        elif op["op"] == "XCONV":
            run_xconv(m, op)
        else:
            run_four_step_pad(m, op)
    assert np.array_equal(m.mem[MULT], keep_mult, equal_nan=True), "the multiplier was written"
    if not inplace:
        assert np.array_equal(m.mem[IN], keep_in, equal_nan=True), "`in` was written"
    for b, arr in m.mem.items():
        assert np.all(arr[sizes[b]:] == CANARY), f"write past the end of buffer {b}"
    got = m.mem[OUT][: nlines * out_len].copy()
    assert not np.isnan(got.view(np.float64)).any(), "an output element was never written (or read NaN)"
    return got, ops


def want(a, M, n, out_len, scaled):
    r = np.fft.ifft(np.fft.fft(a, n=n, axis=-1) * M, axis=-1)[:, :out_len]
    return r if scaled else r * n


def check(got, want_):
    want_ = want_.reshape(-1)
    assert got.shape == want_.shape
    assert np.abs(got - want_).max() <= 1e-11 * max(1.0, np.abs(want_).max())


def pad_cases(n):
    h = max(1, n // 2)
    return [(n, n), (h, min(n, h + 1)), (1, n), (n, 1)]


def run_case(n, in_len, out_len, nlines, seed, shared=True, flags=0, inplace=False, precision=dfft.DOUBLE):
    rng = np.random.default_rng(seed)
    a = rand_c(rng, (nlines, in_len))
    M = rand_c(rng, n if shared else (nlines, n))
    got, ops = simulate(n, in_len, out_len, nlines, a, M, flags, inplace, precision)
    check(got, want(a, M, n, out_len, bool(flags & dfft.SCALE_BACKWARD)))
    for op in ops:
        if op["op"] in ("LINE_CONV_PAD", "XCONV"):
            assert op["shared"] == (1 if shared else 0)
            assert bool(op["do_scale"]) == bool(flags & dfft.SCALE_BACKWARD)
            if op["do_scale"]:
                assert op["scale"] == pytest.approx(1.0 / n, rel=1e-15)
    return ops


@pytest.mark.parametrize("precision", PRECISIONS)
def test_short_path_at_every_tuned_length(precision):
    for n in sorted(dfft.supported_lengths(precision)):
        C = ops_of(n, n, n, 1, precision=precision)[0]["C"]
        nlines = C + 1 if C > 1 else 3            # a partial last tile (for C == 1 every tile is whole)
        for i, (li, lo) in enumerate(pad_cases(n)):
            shared = i % 2 == 0
            flags = dfft.SCALE_BACKWARD if i >= 2 else 0
            ops = run_case(n, li, lo, nlines, n * 13 + i + precision, shared, flags, precision=precision)
            assert [o["op"] for o in ops] == ["LINE_CONV_PAD"]
            op = ops[0]
            assert op["N"] == n and op["W"] == nlines and op["G"] == op["ntiles"] == -(-nlines // C)
            assert op["ia"] == [0, C * li, li, 1] and op["oa"] == [0, C * lo, lo, 1] and op["inv"] == 0
        run_case(n, n, n, nlines, n, shared=False, inplace=True, precision=precision)


# (n, n1, n2, precision): untuned lengths split into two tuned ones -- short untuned lengths, square and oblong splits, 3-, 5- and
# 7-smooth factors -- up to 2^16 points
LONG = [(36, 6, 6, dfft.DOUBLE), (6144, 64, 96, dfft.DOUBLE), (8192, 64, 128, dfft.DOUBLE), (10000, 100, 100, dfft.DOUBLE),
        (2401, 49, 49, dfft.FLOAT), (8192, 64, 128, dfft.FLOAT), (1 << 16, 256, 256, dfft.FLOAT), (1 << 16, 256, 256, dfft.DOUBLE),
        (12288, 96, 128, dfft.FLOAT), (72, 8, 9, dfft.FLOAT)]


@pytest.mark.parametrize("n,n1,n2,precision", LONG)
def test_long_path_splits_and_results(n, n1, n2, precision):
    assert dfft.length_kind(n, precision) != 2
    nlines = 3
    cases = pad_cases(n) + [(n2 - 1, n - 1)]
    for i, (li, lo) in enumerate(cases):
        shared = i % 2 == 1
        flags = dfft.SCALE_BACKWARD if i % 3 == 0 else 0
        ops = run_case(n, li, lo, nlines, n + i + 17 * precision, shared, flags, precision=precision)
        assert [o["op"] for o in ops] == ["XF_TW_PAD", "XCONV", "XB_TW_PAD"]
        a, b, c = ops
        assert (a["N"], b["N"], c["N"]) == (n1, n2, n1), "split"
        assert a["tw_n"] == c["tw_n"] == n and b["tw_n"] == 0
        assert [bufid(o["in"]) for o in ops] == [IN, TEMP, TEMP] and [bufid(o["out"]) for o in ops] == [TEMP, TEMP, OUT]
        assert a["ia"] == [li, a["C"], 1, n2] and a["oa"] == [n, a["C"] * n1, n1, 1] and a["W"] == n2
        assert b["ia"] == b["oa"] == [n, b["C"], 1, n1] and b["W"] == n1
        assert c["ia"] == [n, c["C"] * n1, n1, 1] and c["oa"] == [lo, c["C"], 1, n2] and c["W"] == n2
        assert a["ntiles"] == c["ntiles"] == nlines * a["G"] and b["ntiles"] == nlines * b["G"]
    # in place with lines of the same length in and out, and partial last tiles of every pass (W not a multiple of C)
    run_case(n, n // 2, n // 2, 2, n, inplace=True, precision=precision)


def test_partial_tiles_of_the_long_path():
    ops = ops_of(36, 20, 30, 2)
    assert any(o["W"] % o["C"] for o in ops)
    run_case(36, 20, 30, 2, 1, shared=False)


def test_in_len_equal_out_len_equal_n_is_the_circular_convolution():
    for n in (64, 1000, 8192):
        ops = ops_of(n, n, n, 2)
        rng = np.random.default_rng(n)
        a, M = rand_c(rng, (2, n)), rand_c(rng, n)
        got, _ = simulate(n, n, n, 2, a, M)
        check(got, np.fft.ifft(np.fft.fft(a, axis=-1) * M, axis=-1) * n)
        assert len(ops) == (1 if n <= 4096 else 3)


def test_existing_four_step_splits_are_unchanged():
    # the complex lines plans keep their own split (tests/golden/lines_plan_ops.json pins every one); where a factor lacks a kernel of
    # the padded long path, the padded plan picks another split or none.  At 2^20 both take 1024 x 1024
    fwd = dfft.lines_ops(1 << 20, 1, 1, 1, 1 << 20, 0, dfft.FORWARD)
    pad = ops_of(1 << 20, 1 << 19, 1 << 19, 1)
    assert fwd[0]["N"] == pad[0]["N"] == 1024


def test_empty_batch():
    ops = ops_of(64, 10, 20, 0)
    assert len(ops) == 1 and ops[0]["ntiles"] == 0 and ops[0]["W"] == 0
    ops = ops_of(8192, 10, 20, 0)
    assert len(ops) == 3 and all(o["ntiles"] == 0 for o in ops)


def test_rejections(monkeypatch):
    def c(n, li, lo, nlines=2, flags=0, mult_count=1, precision=dfft.DOUBLE):
        return code(ops_of, n, li, lo, nlines, flags, mult_count, precision)
    assert c(64, 1, 64) == 0 and c(64, 64, 1) == 0 and c(8192, 1, 8192) == 0 and c(64, 3, 5, 4, mult_count=4) == 0
    for li, lo in ((0, 64), (65, 64), (64, 0), (64, 65), (-1, 3), (3, -1)):
        assert c(64, li, lo) == -1, (li, lo)
        assert c(8192, li if li != 65 else 8193, lo if lo != 65 else 8193) == -1, (li, lo)
    assert c(0, 1, 1) == -1 and c(-4, 1, 1) == -1
    assert c(64, 8, 8, nlines=-1) == -1
    assert c(64, 8, 8, precision=7) == -1
    for flags in (dfft.DRY_RUN, dfft.NO_FUSE, dfft.NATURAL_SPECTRUM, dfft.SCALE_BACKWARD | 1, 1 << 31):
        assert c(64, 8, 8, flags=flags) == -1, flags
    for mc in (0, 3, 5, -1):
        assert c(64, 8, 8, nlines=4, mult_count=mc) == -1, mc
    assert c(64, 8, 8, nlines=1 << 31) == -3 and c(64, 8, 8, nlines=(1 << 31) - 1) == 0 and c(64, 8, 8, nlines=1 << 62) == -3
    assert c(8192, 8, 8, nlines=1 << 31) == -3
    for n in (1, 17, 8191, 2 * 8191, 4099 * 2, 1 << 25):     # no tuned entry and no split into two tuned lengths
        assert c(n, 1, 1) == -3, n
    assert c(1 << 24, 1, 1, precision=dfft.FLOAT) == 0 and c(1 << 24, 1, 1) == 0
    assert c(512, 8, 8) == 0
    monkeypatch.setenv("DFFT_VARIANT", "5")                  # an alternate tuning of 512: no padded line-convolution kernel
    assert c(512, 8, 8) == -3
    monkeypatch.delenv("DFFT_VARIANT")
    monkeypatch.setenv("DFFT_GENERIC", "1")                  # run-time-scheduled entries: neither path
    assert c(64, 8, 8) == -3 and c(8192, 8, 8) == -3 and c(36, 8, 8) == -3


def test_null_plan_pointer_is_refused():
    L = dfft.lib()
    assert L.dfft_lines_plan_create_convolve_padded_1d(64, 8, 8, 2, dfft.DOUBLE, 0, None) == -1


def test_python_padded_argument_is_checked():
    with pytest.raises(ValueError):
        dfft.LinesConvolvePlan(one_d=(64, 2), real=True, padded=(8, 8))
    with pytest.raises(ValueError):
        dfft.LinesConvolvePlan(two_d=(16, 16, 2), padded=(8, 8))
    with pytest.raises(ValueError):
        dfft.LinesConvolvePlan(padded=(8, 8))
