"""Every TMA-pipelined kernel (fft_tma.cuh: fft_tma_pass_kernel in modes Z, Y, XF, XB, and fft_tma_fused_zy_kernel) against
a long-double FFT of the exact input (tests/ldfft.py), for every entry of the table in dfft_kernels_tma.cu (pinned in
tests/tma_entries.py) and every mode, by default and under DFFT_TMA=2, which forces every mode.

Metric, against the long-double transform of the values the device was given (the complex64-rounded input in fp32):
rel_l2 = ||got - ref||_2 / ||ref||_2 <= 1.0 * eps * log2(Ntot) and linf = max|got - ref| / rms(ref) <= 4 * eps * log2(Ntot),
eps = 2^-53 (fp64) or 2^-24 (fp32).  numpy's own fp64 FFT measures about 0.14 and 0.6 in these units (16x512x64,
1024x16x64, 8x768x768), so the bounds leave about 7x headroom; a stage whose twiddles are off by 1e-13 fails them
(test_ld_reference.py), where the older bound of 1e-12 * log2(N) relative L-infinity did not.  Every case prints both
ratios ("TMA-RATIO" lines).

Each run uses its own buffers: the output region is prefilled with NaN and fenced by canary elements before and after it,
and the plan executes three times without a refill.  No NaN may survive, the canaries must be bit-unchanged, the three
outputs bit-identical and an out-of-place input unchanged.  The shapes are thin slabs (only the axis under test is long);
tile counts are derived from the device's SM count, since a pass kernel launches min(SMs, tiles) persistent CTAs, each
running a 3-slot ring."""
import faulthandler
import math
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ld_harness  # noqa: E402
import ldfft  # noqa: E402
from ld_harness import bits as _bits, layouts as _layouts, run_fenced  # noqa: E402
from tma_entries import DOUBLE, ENTRIES, FLOAT, MASK_BIT, TMA_LENGTHS, entry_id, modes, thin_shape  # noqa: E402

FWD, BWD = dfft.FORWARD, dfft.BACKWARD
BY = {(e[0], e[1]): e for e in ENTRIES}
REF_FLAGS = dfft.NO_FUSE | dfft.NO_TMA


@pytest.fixture(autouse=True)
def _watchdog():
    # a host-side hang inside libdfft.so cannot be interrupted by a Python-level signal handler
    faulthandler.dump_traceback_later(240, exit=True, file=sys.stderr)
    yield
    faulthandler.cancel_dump_traceback_later()


@pytest.fixture(scope="module", autouse=True)
def _long_double():
    # without an extended long double the reference is no more exact than the fp64 kernels it judges
    assert np.finfo(np.longdouble).eps <= ldfft.LD_EPS_MAX, "np.longdouble is not wider than double: no reference for the fp64 bounds"


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- inputs, references and fenced runs: tests/ld_harness.py ------------------------------------------------------------
def _set_tma(monkeypatch, forced):
    if forced:
        monkeypatch.setenv("DFFT_TMA", "2")
    else:
        monkeypatch.delenv("DFFT_TMA", raising=False)


def check(got, want, prec, ntot, label, linf_scale="rms"):
    return ld_harness.check("TMA-RATIO", got, want, prec, ntot, label, linf_scale)


def _label(entry, mode, forced, what):
    return "%s %s %s %s" % (entry_id(entry), mode, "forced" if forced else "default", what)


# ---- the matrix: every entry, every axis, default and forced -------------------------------------------------------------
AXES = {2: ("Z", "Z"), 1: ("Y", "Y"), 0: ("XF", "XB")}
MATRIX = [(e, axis, forced) for e in ENTRIES for axis in (2, 1, 0) for forced in (False, True)]


@pytest.mark.parametrize("entry,axis,forced", MATRIX, ids=["%s-%s-%s" % (entry_id(e), AXES[a][0][0], "forced" if f else "default") for e, a, f in MATRIX])
def test_pass_mode_against_long_double(entry, axis, forced, monkeypatch):
    _set_tma(monkeypatch, forced)
    N, prec, C, _ = entry
    shape = thin_shape(entry, axis, short=(8, 16))
    ntot = int(np.prod(shape))
    used = modes(entry, forced)
    runs = [(FWD, False, 0), (FWD, True, 0), (BWD, False, 0), (BWD, True, 0), (BWD, False, dfft.SCALE_BACKWARD)]
    for direction, inplace, flags in runs:
        mode = AXES[axis][0 if direction == FWD else 1]
        dev_in, want = _layouts(shape, 1000 + axis, prec, direction, scale=bool(flags))
        got, mask, fused = run_fenced(shape, prec, direction, dev_in, flags=flags, inplace=inplace)
        assert mask == (MASK_BIT[mode] if mode in used else 0), (mode, mask)
        assert not fused
        check(got, want, prec, ntot, _label(entry, mode, forced, "%s%s%s %s" % ("fwd" if direction == FWD else "bwd", " in-place" if inplace else "",
                                                                             " scaled" if flags else "", "x".join(map(str, shape)))))


@pytest.mark.parametrize("forced", [False, True], ids=["default", "forced"])
def test_fused_zy_against_long_double(forced, monkeypatch):
    _set_tma(monkeypatch, forced)
    entry = BY[512, DOUBLE]
    shape = (2, 512, 512)
    dev_in, want = _layouts(shape, 7, DOUBLE, FWD)
    for inplace in (False, True):
        got, mask, fused = run_fenced(shape, DOUBLE, FWD, dev_in, inplace=inplace)
        assert fused and mask == (3 if forced else 2), (fused, mask)
        check(got, want, DOUBLE, dev_in.size, _label(entry, "ZY", forced, "fwd%s 2x512x512" % (" in-place" if inplace else "")))
    for kind in ("delta", "expo"):      # sparse inputs, as in test_sparse_inputs
        dev_in, want = _layouts(shape, 0, DOUBLE, FWD, kind=kind)
        got, _, fused = run_fenced(shape, DOUBLE, FWD, dev_in, repeat=1)
        assert fused
        check(got, want, DOUBLE, dev_in.size, _label(entry, "ZY", forced, "%s fwd 2x512x512" % kind), linf_scale="max")


# ---- tile-count regimes -------------------------------------------------------------------------------------------------
def _smooth(n):
    for p in (2, 3, 5, 7, 11, 13):
        while n % p == 0:
            n //= p
    return n == 1


def _next_smooth(n):
    while not _smooth(n):
        n += 1
    return n


def _ok_len(n):
    return 2 <= n <= 4096 and n not in TMA_LENGTHS


def _regime_shape(entry, axis, tiles):
    """a thin shape whose TMA pass along `axis` has exactly `tiles` tiles (Z: n0*n1/C, Y: n0*n2/C, X: n1*n2/C)"""
    N, _, C, _ = entry
    best = None
    if axis == 2:
        lines = tiles * C
        for a in range(2, lines // 2 + 1):
            if lines % a == 0 and _ok_len(a) and _ok_len(lines // a):
                score = abs(math.log(a / (lines // a)))
                if best is None or score < best[0]:
                    best = (score, (a, lines // a, N))
    else:
        for m in range(1, tiles + 1):
            if tiles % m == 0 and tiles // m >= 2 and _ok_len(m * C) and _ok_len(tiles // m):
                other, n2 = tiles // m, m * C
                score = abs(math.log(other / n2))
                if best is None or score < best[0]:
                    best = (score, (other, N, n2) if axis == 1 else (N, other, n2))
    assert best, (entry, axis, tiles)
    return best[1]


def _tiles(shape, axis, C):
    n0, n1, n2 = shape
    return {2: n0 * n1, 1: n0 * n2, 0: n1 * n2}[axis] // C


# 1 tile (2 for Y and X: an axis of length 1 is not supported), then the smallest 13-smooth count above SMs (every CTA but a
# few runs one tile: a ragged second round), then the smallest above 7 * SMs (every CTA runs >= 7 tiles, so each ring slot and
# its mbarrier phase is used at least twice more).  SMs + 1 itself (133 = 7 * 19 on a 132-SM H100) has no 13-smooth shape.
# The deep regime runs in fp64 only: the tile count is what matters, and an fp32 tile holds twice the points to reference.
REGIME_MODES = [("Z", 256, DOUBLE), ("Y", 1024, DOUBLE), ("XF", 1024, DOUBLE), ("XB", 1024, DOUBLE),
                ("Z", 512, FLOAT), ("Y", 1024, FLOAT), ("XF", 768, FLOAT), ("XB", 768, FLOAT)]
REGIME_CASES = [(m, n, p, r) for r in ("min", "ragged", "deep") for m, n, p in REGIME_MODES if not (r == "deep" and p == FLOAT)]


@pytest.mark.parametrize("mode,N,prec,regime", REGIME_CASES,
                         ids=["%s-%s-%d%s" % (r, m, n, "f64" if p == DOUBLE else "f32") for m, n, p, r in REGIME_CASES])
def test_tile_regimes(mode, N, prec, regime, sms, monkeypatch):
    _set_tma(monkeypatch, False)
    entry = BY[N, prec]
    assert mode in entry[3]
    axis = {"Z": 2, "Y": 1, "XF": 0, "XB": 0}[mode]
    direction = BWD if mode == "XB" else FWD
    C = entry[2]
    if regime == "min":
        tiles = 1 if axis == 2 else 2
    elif regime == "ragged":
        tiles = _next_smooth(sms + 1)
    else:
        tiles = _next_smooth(7 * sms + 1)
    shape = _regime_shape(entry, axis, tiles)
    t = _tiles(shape, axis, C)
    assert t == tiles
    if regime == "min":
        assert t <= 2 < sms
    elif regime == "ragged":
        assert sms < t < 2 * sms and t % sms != 0
    else:
        assert t // sms >= 7 and t % sms != 0
    dev_in, want = _layouts(shape, 2000 + t, prec, direction)
    got, mask, _ = run_fenced(shape, prec, direction, dev_in, flags=dfft.SCALE_BACKWARD if direction == BWD else 0)
    if direction == BWD:
        want = want / np.longdouble(dev_in.size)
    assert mask == MASK_BIT[mode]
    check(got, want, prec, dev_in.size, _label(entry, mode, False, "%s %d tiles on %d SMs %s" % (regime, t, sms, "x".join(map(str, shape)))))


# ---- fallbacks: n2 not a multiple of C keeps the register-staged kernel ---------------------------------------------------
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["f64", "f32"])
@pytest.mark.parametrize("forced", [False, True], ids=["default", "forced"])
def test_fallback_when_n2_is_not_a_multiple_of_c(prec, forced, monkeypatch):
    _set_tma(monkeypatch, forced)
    entry = BY[1024, prec]
    assert 6 % entry[2] != 0
    for axis, direction, mode in ((1, FWD, "Y"), (0, FWD, "XF"), (0, BWD, "XB")):
        shape = (8, 1024, 6) if axis == 1 else (1024, 8, 6)
        dev_in, want = _layouts(shape, 3000 + axis, prec, direction)
        got, mask, _ = run_fenced(shape, prec, direction, dev_in)
        assert mask & MASK_BIT[mode] == 0, mask
        check(got, want, prec, dev_in.size, _label(entry, mode, forced, "fallback n2=6 %s" % "x".join(map(str, shape))))


# ---- sparse inputs: exact spectra that locate index and tile-mapping errors ------------------------------------------------
# L-infinity is taken relative to max|ref| here: the exponential's spectrum is one spike of Ntot, sqrt(Ntot) times its rms, and
# even numpy's fp64 FFT measures ~13 eps log2(Ntot) against that rms at 8x16x512 (for the impulse both scales are 1)
SPARSE = [(e, axis) for e in ENTRIES for axis in (2, 1, 0)]


@pytest.mark.parametrize("entry,axis", SPARSE, ids=["%s-%s" % (entry_id(e), AXES[a][0][0]) for e, a in SPARSE])
def test_sparse_inputs(entry, axis, monkeypatch):
    _set_tma(monkeypatch, True)          # every mode on the TMA kernel
    prec = entry[1]
    shape = thin_shape(entry, axis, short=(8, 16))
    for direction in (FWD, BWD):
        mode = AXES[axis][0 if direction == FWD else 1]
        for kind in ("delta", "expo"):
            dev_in, want = _layouts(shape, 0, prec, direction, kind=kind)
            got, mask, _ = run_fenced(shape, prec, direction, dev_in, repeat=1)
            assert mask == MASK_BIT[mode]
            check(got, want, prec, dev_in.size, _label(entry, mode, True, "%s %s %s" % (kind, "fwd" if direction == FWD else "bwd", "x".join(map(str, shape)))),
                  linf_scale="max")


# ---- fused ZY: lag sweep bit for bit, natural spectrum ----------------------------------------------------------------------
@pytest.mark.parametrize("n0", [5, 24])
def test_fused_zy_lag_sweep_is_bitwise_the_register_staged_sweeps(n0, monkeypatch):
    _set_tma(monkeypatch, False)
    shape = (n0, 512, 512)
    rng = np.random.default_rng(n0)
    x = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).reshape(-1)
    ref, _, fused = run_fenced(shape, DOUBLE, FWD, x, flags=REF_FLAGS, repeat=1)
    assert not fused
    for lag in (1, 2, None, n0 + 5):
        if lag is None:
            monkeypatch.delenv("DFFT_LAG", raising=False)
        else:
            monkeypatch.setenv("DFFT_LAG", str(lag))
        got, _, fused = run_fenced(shape, DOUBLE, FWD, x)
        assert fused
        assert np.array_equal(_bits(got), _bits(ref)), ("lag", lag)


@pytest.mark.parametrize("direction", [FWD, BWD], ids=["fwd", "bwd"])
def test_natural_spectrum_16x512x512(direction, monkeypatch):
    _set_tma(monkeypatch, False)
    shape = (16, 512, 512)
    dev_in, want = _layouts(shape, 16, DOUBLE, direction, natural=True)
    got, _, fused = run_fenced(shape, DOUBLE, direction, dev_in, flags=dfft.NATURAL_SPECTRUM)
    assert fused == (direction == FWD)
    check(got, want, DOUBLE, dev_in.size, _label(BY[512, DOUBLE], "ZY" if direction == FWD else "Y", False, "natural %s 16x512x512" % ("fwd" if direction == FWD else "bwd")))


# ---- regressions: DFFT_TMA=2 on mixed lengths, plans of different lengths, unaligned complex64 buffers ----------------------
MIXED = [((1024, 4, 512), 1 | 4), ((1024, 512, 8), 2 | 4), ((512, 256, 16), 2 | 4)]   # (shape, tma_mask in either direction)


@pytest.mark.parametrize("shape,want_mask", MIXED, ids=["x".join(map(str, m[0])) for m in MIXED])
def test_forced_mixed_lengths_keep_each_axis_entry(shape, want_mask, monkeypatch):
    """under DFFT_TMA=2 each axis runs the kernel of its own length (Z at 512 and X at 1024; Y at 512 and X at 1024; Y at 256
    and X at 512)"""
    _set_tma(monkeypatch, True)
    for direction in (FWD, BWD):
        dev_in, want = _layouts(shape, 4000, DOUBLE, direction)
        got, mask, _ = run_fenced(shape, DOUBLE, direction, dev_in, repeat=2)
        assert mask == want_mask
        check(got, want, DOUBLE, dev_in.size, "mixed forced %s %s" % ("fwd" if direction == FWD else "bwd", "x".join(map(str, shape))))


def test_two_plans_of_different_lengths_executed_alternately(monkeypatch):
    _set_tma(monkeypatch, True)
    shapes = [(2, 512, 16), (1024, 2, 16)]     # Y at 512 (C = 8), then X at 1024 (C = 4), created on one thread
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    ins, outs, wants, plans = [], [], [], []
    for k, shape in enumerate(shapes):
        dev_in, want = _layouts(shape, 5000 + k, DOUBLE, FWD)
        ins.append(torch.from_numpy(dev_in).to(dev))
        outs.append(torch.full_like(ins[-1], complex(float("nan"), float("nan"))))
        wants.append(want)
    torch.cuda.synchronize(dev)
    for k, shape in enumerate(shapes):
        plans.append(dfft.fft_mpi_plan_dft_c2c_3d(*shape, ins[k].data_ptr(), outs[k].data_ptr(), None, 0, 1, FWD, DOUBLE, 0))
    assert [p.tma_mask for p in plans] == [2, 4]
    try:
        first = [None, None]
        for _ in range(2):
            for k, p in enumerate(plans):
                p.execute()
                p.synchronize()
                got = outs[k].cpu().numpy()
                if first[k] is None:
                    first[k] = got
                    check(got, wants[k], DOUBLE, got.size, "two plans forced %s" % "x".join(map(str, shapes[k])))
                else:
                    assert np.array_equal(_bits(got), _bits(first[k])), k
    finally:
        for p in plans:
            p.destroy()


@pytest.mark.parametrize("inplace", [False, True], ids=["out-of-place", "in-place"])
def test_complex64_output_view_at_odd_element_offset(inplace, monkeypatch):
    """bufferDev2 8 bytes off 16-byte alignment: the plan keeps every pass on the register-staged kernels, and the result is
    as exact as ever, with the canaries on both sides intact"""
    for forced in (False, True):
        _set_tma(monkeypatch, forced)
        entry = BY[512, FLOAT]
        for axis in (1, 0, 2):
            shape = thin_shape(entry, axis, short=(8, 16))
            for direction in (FWD, BWD):
                dev_in, want = _layouts(shape, 6000 + axis, FLOAT, direction)
                got, mask, fused = run_fenced(shape, FLOAT, direction, dev_in, inplace=inplace, offset=1)
                assert mask == 0 and not fused
                check(got, want, FLOAT, dev_in.size, "512f32 %s offset-1 %s %s %s" % ("forced" if forced else "default", "in-place" if inplace else "out-of-place",
                                                                                      "fwd" if direction == FWD else "bwd", "x".join(map(str, shape))))


def test_complex128_buffer_off_16_byte_alignment_is_rejected():
    dev = torch.device("cuda", 0)
    buf = torch.zeros(2 * 8 * 512 * 16 + 2, dtype=torch.complex128, device=dev)
    with pytest.raises(dfft.DfftError, match="16-byte aligned"):
        dfft.fft_mpi_plan_dft_c2c_3d(8, 512, 16, buf.data_ptr(), buf.data_ptr() + 8 + 16 * 8 * 512 * 16, None, 0, 1, FWD)
