"""CPU tests of the real zero-padded 1-D convolve lines plans (dfft_lines_plan_create_convolve_padded_r2c_1d) without a GPU.

dfft_debug_lines_conv_padded_r2c_1d_ops records the passes one execute launches: "LINE_CONV_PAD_R2C" (short path), or
"XF_TW_PAD_R2C", "XCONV_R2C" and "XB_TW_PAD_C2R" (long path, four-step over line pairs z = a + i b).  The interpreters below give
the records their meaning, including the mirror-adjacent column order of the temporary (pos) and the mirror partner of each bin
in the middle pass, and the result is compared with irfft(rfft(a, n) * m, n)[:, :out_len] * n.  Every buffer starts NaN-filled
with canaries right past its end, so a read past nlines * in_len, an output element left unwritten or a write past
nlines * out_len shows up; `in` (when distinct) and the multiplier must come back unchanged.  The kernels' arithmetic is checked
on the GPU by test_gpu_lines_conv_padded_r2c.py."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_dry_run import IN, OUT
from test_lines_conv_dry_run import MULT, TEMP, ConvMachine, code, rand_c
from test_lines_conv_padded_dry_run import ops_of as complex_ops_of
from test_r2c_dry_run import real_view
from test_real_lines_dry_run import CANARY, bufid

PRECISIONS = [dfft.DOUBLE, dfft.FLOAT]


def pos(k1, n1):
    """position of column k1 inside a row of the temporary: mirror columns k1 and n1 - k1 side by side"""
    if n1 % 2 == 0:
        if k1 == 0:
            return 0
        if 2 * k1 == n1:
            return 1
        return 2 * k1 if 2 * k1 < n1 else 2 * (n1 - k1) + 1
    if k1 == 0:
        return n1 - 1
    return 2 * k1 - 2 if 2 * k1 < n1 else 2 * (n1 - k1) - 1


def test_pos_is_a_permutation_that_pairs_mirrors():
    for n1 in list(range(2, 70)) + [125, 243, 1000, 4096]:
        p = [pos(k, n1) for k in range(n1)]
        assert sorted(p) == list(range(n1)), n1
        inv = {q: k for k, q in enumerate(p)}
        for q in range(0, n1, 2):   # every aligned position pair holds a mirror pair or self-mirrored columns
            ks = [inv[x] for x in (q, q + 1) if x < n1]
            for k in ks:
                assert (n1 - k) % n1 in ks, (n1, q, ks)


def run_line_conv_pad_r2c(m, op):
    """LINE_CONV_PAD_R2C: pair tile*C + c, line h of the pair at base + tile*SB + c*cs + h*pair + e*es on each side (reals); points
    e < in_len are read, the rest are zero; rfft, the product with the line's multiplier (nzh points), irfft (unnormalised), the
    optional scale; points e < out_len are stored"""
    N, C, W, H = op["N"], op["C"], op["W"], op["nzh"]
    assert H == N // 2 + 1 and W == op["lines"]
    _, SBi, csi, esi = op["ia"]
    _, SBo, cso, eso = op["oa"]
    ldi, ldo = op["pair"]
    li, lo = op["in_len"], op["out_len"]
    src, soff = real_view(m, op["in"], True)
    dst, doff = real_view(m, op["out"], True)
    mul, moff = m.view(op["mult"])
    ei, eo, j = np.arange(li), np.arange(lo), np.arange(H)
    staged = []
    for tile in range(op["ntiles"]):
        for c in range(C):
            for h in range(2):
                line = 2 * (tile * C + c) + h
                if line >= W:
                    continue
                v = np.zeros(N)
                v[:li] = src[soff + tile * SBi + c * csi + h * ldi + ei * esi]
                x = np.fft.irfft(np.fft.rfft(v) * mul[moff + (0 if op["shared"] else line * H) + j], n=N) * N
                if op["do_scale"]:
                    x = x * op["scale"]
                staged.append((tile, c, h, x))
    for tile, c, h, x in staged:   # every line is read before any is stored: in place is allowed when in_len == out_len
        dst[doff + tile * SBo + c * cso + h * ldo + eo * eso] = x[:lo]


def run_xf_tw_pad_r2c(m, op):
    """XF_TW_PAD_R2C: per line pair a (ia.SA reals apart, the second line `pair[0]` further) and column col = b*C + c < W: point e
    at offset b*SB + c*cs + e*es inside each line, read where that offset is < in_len (zero otherwise, and the second line is zero
    when 2a + 1 >= lines), as z = x + i y; FFT; twiddle e^{-2 pi i col*k / tw_n}; point k stored through the output map at
    position pos(k, N) of the row"""
    N, C, G, W, tw = op["N"], op["C"], op["G"], op["W"], op["tw_n"]
    SAi, SBi, csi, esi = op["ia"]
    SAo, SBo, cso, eso = op["oa"]
    ldi, ldo = op["pair"]
    assert op["tstore"] == 1 and op["inv"] == 0 and not op["do_scale"] and ldo == 0
    src, soff = real_view(m, op["in"], True)
    dst, doff = m.view(op["out"])
    e = np.arange(N)
    p = np.array([pos(k, N) for k in range(N)])
    for tile in range(op["ntiles"]):
        a, b = divmod(tile, G)
        for c in range(C):
            col = b * C + c
            if col >= W:
                continue
            rel = b * SBi + c * csi + e * esi
            ok = rel < op["in_len"]
            v = np.zeros(N, dtype=np.complex128)
            v.real[ok] = src[soff + a * SAi + rel[ok]]
            if 2 * a + 1 < op["lines"]:
                v.imag[ok] = src[soff + a * SAi + ldi + rel[ok]]
            x = np.fft.fft(v) * np.exp(-2j * np.pi * ((col * e) % tw) / tw)
            dst[doff + a * SAo + b * SBo + c * cso + p * eso] = x


def run_xconv_r2c(m, op):
    """XCONV_R2C: per line pair a and tile b of column positions (W = n1 of them): column position cp holds column k1 with
    pos(k1, n1) = cp; FFT along N = n2, so that element k2 of column k1 is Z[e], e = k1 + n1*k2, n = n1*n2.  The partner Z[n - e]
    must lie in the same tile.  With j = min(e, n - e), F = Z[j], G = Z[n - j]: A = (F + conj G)/2, B = (F - conj G)/2i, A' = A
    ma[j], B' = B mb[j] (mb = 0 for a missing second line), Im A' = Im B' = 0 at j = 0 and 2j = n, optional scale; Z'[e] = A' + i B'
    for 2e <= n, conj A' + i conj B' above; inverse FFT along n2 (unnormalised), stored in place through the output map"""
    N, C, G, W = op["N"], op["C"], op["G"], op["W"]
    n1, n = W, W * N
    H = op["nzh"]
    assert H == n // 2 + 1 and op["ia"] == op["oa"]
    SA, SB, cs, es = op["ia"]
    src, soff = m.view(op["in"])
    dst, doff = m.view(op["out"])
    mul, moff = m.view(op["mult"])
    inv = {pos(k, n1): k for k in range(n1)}
    k2 = np.arange(N)
    staged = []
    for tile in range(op["ntiles"]):
        a, b = divmod(tile, G)
        Z = {}
        for c in range(C):
            if b * C + c < W:
                Z[inv[b * C + c]] = (c, np.fft.fft(src[soff + a * SA + b * SB + c * cs + k2 * es]))
        ma = mul[moff + (0 if op["shared"] else 2 * a * H) + np.arange(H)]
        mb = mul[moff + (0 if op["shared"] else (2 * a + 1) * H) + np.arange(H)] if 2 * a + 1 < op["lines"] else np.zeros(H)
        for k1, (c, z) in Z.items():
            e = k1 + n1 * k2
            pe = (n - e) % n
            pk1 = (n1 - k1) % n1
            assert pk1 in Z, ("the mirror column is not in the tile", k1, pk1)
            w = Z[pk1][1][pe // n1]
            mirror = 2 * e > n
            j = np.where(mirror, n - e, e)
            F, Gv = np.where(mirror, w, z), np.where(mirror, z, w)
            A = (F + np.conj(Gv)) / 2 * ma[j]
            B = (F - np.conj(Gv)) / 2j * mb[j]
            edge = (j == 0) | (2 * j == n)
            A = np.where(edge, A.real, A)
            B = np.where(edge, B.real, B)
            if op["do_scale"]:
                A, B = A * op["scale"], B * op["scale"]
            Zp = np.where(mirror, np.conj(A) + 1j * np.conj(B), A + 1j * B)
            staged.append((a, b, c, np.fft.ifft(Zp) * N))
    for a, b, c, x in staged:
        dst[doff + a * SA + b * SB + c * cs + k2 * es] = x


def run_xb_tw_pad_c2r(m, op):
    """XB_TW_PAD_C2R: per line pair a and row col = b*C + c < W: point k of the row read at position pos(k, N) through the input
    map; twiddle e^{+2 pi i col*k / tw_n}; inverse FFT (unnormalised); point j1 at offset b*SB + c*cs + j1*es inside the output
    lines (oa.SA reals apart), stored where that offset is < out_len: Re to line 2a, Im to line 2a + 1 (`pair[1]` further) when
    2a + 1 < lines"""
    N, C, G, W, tw = op["N"], op["C"], op["G"], op["W"], op["tw_n"]
    SAi, SBi, csi, esi = op["ia"]
    SAo, SBo, cso, eso = op["oa"]
    ldi, ldo = op["pair"]
    assert op["tstore"] == 0 and op["inv"] == 1 and not op["do_scale"] and ldi == 0
    src, soff = m.view(op["in"])
    dst, doff = real_view(m, op["out"], True)
    e = np.arange(N)
    p = np.array([pos(k, N) for k in range(N)])
    staged = []
    for tile in range(op["ntiles"]):
        a, b = divmod(tile, G)
        for c in range(C):
            col = b * C + c
            if col >= W:
                continue
            v = src[soff + a * SAi + b * SBi + c * csi + p * esi]
            x = np.fft.ifft(v * np.exp(2j * np.pi * ((col * e) % tw) / tw)) * N
            staged.append((a, b, c, x))
    for a, b, c, x in staged:
        rel = b * SBo + c * cso + e * eso
        ok = rel < op["out_len"]
        dst[doff + a * SAo + rel[ok]] = x.real[ok]
        if 2 * a + 1 < op["lines"]:
            dst[doff + a * SAo + ldo + rel[ok]] = x.imag[ok]


RUN = {"LINE_CONV_PAD_R2C": run_line_conv_pad_r2c, "XF_TW_PAD_R2C": run_xf_tw_pad_r2c, "XCONV_R2C": run_xconv_r2c,
       "XB_TW_PAD_C2R": run_xb_tw_pad_c2r}


def ops_of(n, in_len, out_len, nlines, flags=0, mult_count=1, precision=dfft.DOUBLE):
    return dfft.lines_conv_padded_1d_ops(n, in_len, out_len, nlines, precision, flags, mult_count, real=True)


def simulate(n, in_len, out_len, nlines, a, M, flags=0, inplace=False, precision=dfft.DOUBLE):
    """a: [nlines][in_len] real input; M: the multiplier, [n/2+1] (shared) or [nlines][n/2+1]"""
    mult_count = 1 if M.ndim == 1 else nlines
    reals = {IN: nlines * in_len, OUT: nlines * out_len}
    sizes = {IN: -(-reals[IN] // 2), OUT: -(-reals[OUT] // 2), MULT: (n // 2 + 1) * mult_count, TEMP: -(-nlines // 2) * n}
    m = ConvMachine(sizes, inplace)
    for b, r in reals.items():   # the real buffers' canaries start right after their last real
        m.mem[b].view(np.float64)[r:] = CANARY
    m.mem[IN].view(np.float64)[: a.size] = a.reshape(-1)
    m.mem[MULT][: M.size] = M.reshape(-1)
    keep_in, keep_mult = m.mem[IN].copy(), m.mem[MULT].copy()
    ops = ops_of(n, in_len, out_len, nlines, flags, mult_count, precision)
    for op in ops:
        assert bufid(op["out"]) != MULT and (inplace or bufid(op["out"]) != IN), ("a pass writes a read-only buffer", op["op"])
        assert (op["in_len"], op["out_len"], op["lines"]) == (in_len, out_len, nlines)
        RUN[op["op"]](m, op)
    assert np.array_equal(m.mem[MULT], keep_mult, equal_nan=True), "the multiplier was written"
    if not inplace:
        assert np.array_equal(m.mem[IN], keep_in, equal_nan=True), "`in` was written"
    for b, arr in m.mem.items():
        tail = arr.view(np.float64)[reals[b]:] if b in reals else arr[sizes[b]:]
        assert np.all(tail == CANARY), f"write past the end of buffer {b}"
    got = m.mem[OUT].view(np.float64)[: nlines * out_len].copy()
    assert not np.isnan(got).any(), "an output element was never written (or read NaN)"
    return got, ops


def want(a, M, n, out_len, scaled):
    r = np.fft.irfft(np.fft.rfft(a, n=n, axis=-1) * M, n=n, axis=-1)[:, :out_len]
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
    a = rng.standard_normal((nlines, in_len))
    M = rand_c(rng, n // 2 + 1 if shared else (nlines, n // 2 + 1))
    got, ops = simulate(n, in_len, out_len, nlines, a, M, flags, inplace, precision)
    check(got, want(a, M, n, out_len, bool(flags & dfft.SCALE_BACKWARD)))
    for op in ops:
        if op["op"] in ("LINE_CONV_PAD_R2C", "XCONV_R2C"):
            assert op["shared"] == (1 if shared else 0) and bufid(op["mult"]) == MULT
            assert bool(op["do_scale"]) == bool(flags & dfft.SCALE_BACKWARD)
            if op["do_scale"]:
                assert op["scale"] == pytest.approx(1.0 / n, rel=1e-15)
    return ops


@pytest.mark.parametrize("precision", PRECISIONS)
def test_short_path_at_every_tuned_length(precision):
    for n in sorted(dfft.supported_lengths(precision)):
        if n < 2:
            continue
        C = ops_of(n, n, n, 1, precision=precision)[0]["C"]
        nlines = 2 * C + 1                        # an odd line count (the last pair has no second line), a partial last tile
        for i, (li, lo) in enumerate(pad_cases(n)):
            shared = i % 2 == 0
            flags = dfft.SCALE_BACKWARD if i >= 2 else 0
            ops = run_case(n, li, lo, nlines, n * 13 + i + precision, shared, flags, precision=precision)
            assert [o["op"] for o in ops] == ["LINE_CONV_PAD_R2C"]
            op = ops[0]
            assert op["N"] == n and op["W"] == nlines and op["G"] == op["ntiles"] == -(-(-(-nlines // 2)) // C)
            assert op["ia"] == [0, 2 * C * li, 2 * li, 1] and op["oa"] == [0, 2 * C * lo, 2 * lo, 1] and op["inv"] == 0
            assert op["pair"] == [li, lo] and op["nzh"] == n // 2 + 1
            assert (bufid(op["in"]), bufid(op["out"])) == (IN, OUT)
        run_case(n, n, n, nlines, n, shared=False, inplace=True, precision=precision)


# (n, n1, n2, precision): both factors even, n1 even and n2 odd, n1 odd and n2 even, both odd, a short untuned length
LONG = [(6144, 64, 96, dfft.DOUBLE), (8192, 64, 128, dfft.DOUBLE), (8192, 64, 128, dfft.FLOAT), (1 << 16, 256, 256, dfft.FLOAT),
        (72, 8, 9, dfft.FLOAT), (16000, 125, 128, dfft.DOUBLE), (2401, 49, 49, dfft.FLOAT), (36, 6, 6, dfft.DOUBLE)]


@pytest.mark.parametrize("n,n1,n2,precision", LONG)
def test_long_path_splits_and_results(n, n1, n2, precision):
    assert dfft.length_kind(n, precision) != 2
    nlines = 3
    rows = 2
    cases = pad_cases(n) + [(n2 - 1, n - 1)]
    for i, (li, lo) in enumerate(cases):
        shared = i % 2 == 1
        flags = dfft.SCALE_BACKWARD if i % 3 == 0 else 0
        ops = run_case(n, li, lo, nlines, n + i + 17 * precision, shared, flags, precision=precision)
        assert [o["op"] for o in ops] == ["XF_TW_PAD_R2C", "XCONV_R2C", "XB_TW_PAD_C2R"]
        a, b, c = ops
        assert (a["N"], b["N"], c["N"]) == (n1, n2, n1), "split"
        cx = complex_ops_of(n, li, lo, nlines, precision=precision)
        assert [o["N"] for o in cx] == [n1, n2, n1], "the complex padded plan's split"
        assert [o["C"] for o in cx] == [a["C"], b["C"], c["C"]] and b["C"] % 2 == 0
        assert a["tw_n"] == c["tw_n"] == n and b["tw_n"] == 0
        assert [bufid(o["in"]) for o in ops] == [IN, TEMP, TEMP] and [bufid(o["out"]) for o in ops] == [TEMP, TEMP, OUT]
        assert a["ia"] == [2 * li, a["C"], 1, n2] and a["oa"] == [n, a["C"] * n1, n1, 1] and a["W"] == n2 and a["pair"] == [li, 0]
        assert b["ia"] == b["oa"] == [n, b["C"], 1, n1] and b["W"] == n1 and b["nzh"] == n // 2 + 1 and "pair" not in b
        assert c["ia"] == [n, c["C"] * n1, n1, 1] and c["oa"] == [2 * lo, c["C"], 1, n2] and c["W"] == n2 and c["pair"] == [0, lo]
        assert a["ntiles"] == c["ntiles"] == rows * a["G"] and b["ntiles"] == rows * b["G"]
        assert "mult" not in a and "mult" not in c
    # in place with lines of the same length in and out, an even line count, partial last tiles of every pass
    run_case(n, n // 2, n // 2, 2, n, inplace=True, precision=precision)


def test_sixteen_thousand_splits_with_the_smaller_odd_n1():
    # 16000 = 125 * 128 = 128 * 125: equally square, the tie goes to the smaller n1
    ops = ops_of(16000, 8000, 8000, 1)
    assert [o["N"] for o in ops] == [125, 128, 125]


def test_partial_tiles_of_the_long_path():
    ops = ops_of(36, 20, 30, 5)
    assert any(o["W"] % o["C"] for o in ops)
    run_case(36, 20, 30, 5, 1, shared=False)


def test_in_len_equal_out_len_equal_n_is_the_circular_convolution():
    for n in (64, 1000, 8192):
        rng = np.random.default_rng(n)
        a, M = rng.standard_normal((3, n)), rand_c(rng, n // 2 + 1)
        got, ops = simulate(n, n, n, 3, a, M)
        check(got, np.fft.irfft(np.fft.rfft(a, axis=-1) * M, n=n, axis=-1) * n)
        assert len(ops) == (1 if n <= 4096 else 3)


def test_imaginary_parts_of_the_edge_bins_are_ignored():
    for n, nlines in ((64, 3), (8192, 3), (2401, 2), (72, 3)):
        rng = np.random.default_rng(n)
        a, M = rng.standard_normal((nlines, n // 3)), rand_c(rng, (nlines, n // 2 + 1))
        got, _ = simulate(n, n // 3, n // 2, nlines, a, M)
        M2 = M.copy()
        M2[:, 0] += 3.5j
        if n % 2 == 0:
            M2[:, n // 2] -= 1.25j
        got2, _ = simulate(n, n // 3, n // 2, nlines, a, M2)
        assert np.array_equal(got, got2)


def test_empty_batch():
    ops = ops_of(64, 10, 20, 0)
    assert len(ops) == 1 and ops[0]["ntiles"] == 0 and ops[0]["W"] == 0
    ops = ops_of(8192, 10, 20, 0)
    assert len(ops) == 3 and all(o["ntiles"] == 0 for o in ops)


def test_rejections(monkeypatch):
    def c(n, li, lo, nlines=2, flags=0, mult_count=1, precision=dfft.DOUBLE):
        return code(ops_of, n, li, lo, nlines, flags, mult_count, precision)
    assert c(64, 1, 64) == 0 and c(64, 64, 1) == 0 and c(8192, 1, 8192) == 0 and c(64, 3, 5, 5, mult_count=5) == 0
    assert c(4, 1, 4) == 0 and c(2, 1, 2) == -3                 # 2 points: neither a tuned length nor a split
    for li, lo in ((0, 64), (65, 64), (64, 0), (64, 65), (-1, 3), (3, -1)):
        assert c(64, li, lo) == -1, (li, lo)
        assert c(8192, li if li != 65 else 8193, lo if lo != 65 else 8193) == -1, (li, lo)
    assert c(0, 1, 1) == -1 and c(-4, 1, 1) == -1
    assert c(1, 1, 1) == -3                                  # a real convolution needs at least 2 points
    assert c(64, 8, 8, nlines=-1) == -1
    assert c(64, 8, 8, precision=7) == -1
    for flags in (dfft.DRY_RUN, dfft.NO_FUSE, dfft.NATURAL_SPECTRUM, dfft.SCALE_BACKWARD | 1, 1 << 31):
        assert c(64, 8, 8, flags=flags) == -1, flags
    for mc in (0, 3, 5, -1):
        assert c(64, 8, 8, nlines=4, mult_count=mc) == -1, mc
    assert c(64, 8, 8, nlines=1 << 31) == -3 and c(64, 8, 8, nlines=(1 << 31) - 1) == 0 and c(64, 8, 8, nlines=1 << 62) == -3
    assert c(8192, 8, 8, nlines=1 << 31) == -3
    for n in (17, 8191, 2 * 8191, 4099 * 2, 1 << 25):        # no tuned entry and no split into two tuned lengths
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
    assert L.dfft_lines_plan_create_convolve_padded_r2c_1d(64, 8, 8, 2, dfft.DOUBLE, 0, None) == -1


def test_python_real_padded_argument_is_checked():
    with pytest.raises(ValueError):
        dfft.LinesConvolvePlan(one_d=(64, 2), real_padded=(8, 8), padded=(8, 8))
    with pytest.raises(ValueError):
        dfft.LinesConvolvePlan(one_d=(64, 2), real_padded=(8, 8), real=True)
    with pytest.raises(ValueError):
        dfft.LinesConvolvePlan(two_d=(16, 16, 2), real_padded=(8, 8))
    with pytest.raises(ValueError):
        dfft.LinesConvolvePlan(real_padded=(8, 8))
