"""Every register-staged and generic FFT kernel one GPU can reach, against a long-double FFT of the exact input (tests/ldfft.py),
with the bounds of test_gpu_tma_matrix.py and no per-case loosening: rel_l2 <= 1.0 * eps * log2(Ntot) and max error / rms(ref)
<= 4 * eps * log2(Ntot) (max error / max|ref| for the structured inputs), eps = 2^-53 (fp64) or 2^-24 (fp32).

- fft_tile_kernel: every default entry of dfft_kernels_f64.cu / dfft_kernels_f32.cu (pinned in tests/tile_entries.py) along every
  axis of a thin slab, flags NO_TMA | NO_FUSE: PK_Z, PK_Y, PK_XF and PK_XB forward, backward, in place and scaled, and on the X
  axis the natural spectrum (x_natural: PK_Y with the X length's strided schedule).  The short axes (9, 10) leave a ragged last
  tile wherever C > 2.  Then a delta at the last element and an exponential at bin N - 1 of the long axis, complex64 outputs at
  an odd element offset (default flags: no TMA kernel may run there), and tile counts at which every CTA of the persistent grid
  runs several tiles (against scipy's fp64 FFT, whose own error of about 0.14 / 0.6 in these units is included).
- fft_fused2_kernel (FK_ZY forward, FK_YZ backward) of every entry on (3, N, N): bit-identical to the two sweeps it replaces,
  which carries the bounds over; (3, 64, 64) is also checked against long double directly.  Where an entry has no such kernel
  (tile_entries.NOT_FUSED: its roles do not fit in shared memory together) FORCE_FUSE must keep the two sweeps.
- fft_generic_kernel: lengths that cover radices 2 .. 13 and the shared-memory limits (6400 fp64, 12800 fp32), and DFFT_GENERIC=1
  on tuned lengths, through the same thin-slab runs.
- The lines engine: the four-step long-line plan (PK_XF_TW with its sincospi twiddle epilogue, then PK_Y) and a 2-D LinesPlan,
  against a long-double FFT along the transformed axes (Ntot = points per transform).

Outputs are NaN-prefilled and fenced by canaries, plans execute more than once with bit-identical results, and an out-of-place
input must be unchanged (tests/ld_harness.py).  Every case prints a "TILE-RATIO" line; test_zz_report_worst_ratios prints the
worst per family and precision ("TILE-WORST")."""
import faulthandler
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ld_harness  # noqa: E402
import ldfft  # noqa: E402
from ld_harness import CDT, EPS, bits, layouts, ratios64, run_fenced, run_lines  # noqa: E402
from tile_entries import DOUBLE, ENTRIES, FLOAT, NOT_FUSED, entry_id, lengths, thin_shape, threads  # noqa: E402

FWD, BWD = dfft.FORWARD, dfft.BACKWARD
REF_FLAGS = dfft.NO_TMA | dfft.NO_FUSE
PASS = {2: ("Z", "Z"), 1: ("Y", "Y"), 0: ("XF", "XB")}
RUNS = [(FWD, False, 0), (FWD, True, 0), (BWD, False, 0), (BWD, True, 0), (BWD, False, dfft.SCALE_BACKWARD)]
PN = {DOUBLE: "f64", FLOAT: "f32"}
WORST = {}


@pytest.fixture(autouse=True)
def _watchdog(monkeypatch):
    # a host-side hang inside libdfft.so cannot be interrupted by a Python-level signal handler
    faulthandler.dump_traceback_later(240, exit=True, file=sys.stderr)
    for var in ("DFFT_TMA", "DFFT_GENERIC", "DFFT_FUSE", "DFFT_VARIANT", "DFFT_LAG"):
        monkeypatch.delenv(var, raising=False)
    yield
    faulthandler.cancel_dump_traceback_later()


@pytest.fixture(scope="module", autouse=True)
def _long_double():
    assert np.finfo(np.longdouble).eps <= ldfft.LD_EPS_MAX, "np.longdouble is not wider than double: no reference for the fp64 bounds"


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _note(family, prec, r):
    w = WORST.get((family, prec), (0.0, 0.0))
    WORST[family, prec] = (max(w[0], r[0]), max(w[1], r[1]))


def check(family, got, want, prec, ntot, label, linf_scale="rms"):
    r = ld_harness.check("TILE-RATIO", got, want, prec, ntot, "%s %s" % (family, label), linf_scale)
    _note(family, prec, r)


def xs(shape):
    return "x".join(map(str, shape))


# ---- thin slabs: every pass of one axis ----------------------------------------------------------------------------------
def run_axis(n, prec, axis, family=None):
    """forward, forward in place, backward, backward in place, backward scaled (and on the X axis the natural spectrum both
    ways) of the thin slab whose `axis` has length n, with NO_TMA | NO_FUSE: no TMA kernel, no fused kernel, three launches"""
    shape = thin_shape(n, axis)
    ntot = int(np.prod(shape))
    runs = [(d, ip, s, False) for d, ip, s in RUNS] + ([(FWD, False, 0, True), (BWD, False, 0, True)] if axis == 0 else [])
    for direction, inplace, scale, natural in runs:
        dev_in, want = layouts(shape, 1000 + axis, prec, direction, natural=natural, scale=bool(scale))
        info = {}
        got, mask, fused = run_fenced(shape, prec, direction, dev_in, flags=REF_FLAGS | scale | (dfft.NATURAL_SPECTRUM if natural else 0),
                                      inplace=inplace, info=info)
        assert mask == 0 and not fused and info["launches"] == 3, (mask, fused, info)
        mode = "natural-X" if natural else PASS[axis][direction == BWD]
        check(family or mode, got, want, prec, ntot, "%d%s %s %s%s%s %s" % (n, PN[prec], mode, "fwd" if direction == FWD else "bwd",
                                                                         " in-place" if inplace else "", " scaled" if scale else "", xs(shape)))


MATRIX = [(e, axis) for e in ENTRIES for axis in (2, 1, 0)]
MATRIX_IDS = ["%s-%s" % (entry_id(e), PASS[a][0][0]) for e, a in MATRIX]


@pytest.mark.parametrize("entry,axis", MATRIX, ids=MATRIX_IDS)
def test_register_staged_pass_against_long_double(entry, axis):
    run_axis(entry[0], entry[1], axis)


# ---- structured inputs: exact spectra that locate index, twiddle-sign and tile-mapping errors --------------------------------
# L-infinity relative to max|ref|: the exponential's spectrum is one spike, sqrt(Ntot) times its rms
@pytest.mark.parametrize("entry,axis", MATRIX, ids=MATRIX_IDS)
def test_structured_inputs(entry, axis):
    n, prec = entry[0], entry[1]
    shape = thin_shape(n, axis)
    for direction in (FWD, BWD):
        for kind in ("delta", "expo"):
            dev_in, want = layouts(shape, 0, prec, direction, kind=kind, axis=axis if kind == "expo" else None)
            got, mask, _ = run_fenced(shape, prec, direction, dev_in, flags=REF_FLAGS, repeat=1)
            assert mask == 0
            check("structured", got, want, prec, dev_in.size, "%s %s %s %s" % (entry_id(entry), kind, "fwd" if direction == FWD else "bwd", xs(shape)),
                  linf_scale="max")


# ---- complex64 output at an odd element offset: default flags, register-staged kernels only --------------------------------
F32 = [e for e in ENTRIES if e[1] == FLOAT]


@pytest.mark.parametrize("entry", F32, ids=[entry_id(e) for e in F32])
def test_fp32_output_at_odd_complex64_offset(entry):
    n = entry[0]
    for axis in (2, 0):
        shape = thin_shape(n, axis)
        for direction in (FWD, BWD):
            dev_in, want = layouts(shape, 1000 + axis, FLOAT, direction)
            got, mask, _ = run_fenced(shape, FLOAT, direction, dev_in, offset=1)
            assert mask == 0, mask
            check("offset-1", got, want, FLOAT, dev_in.size, "%s %s %s %s" % (entry_id(entry), PASS[axis][direction == BWD], "fwd" if direction == FWD else "bwd", xs(shape)))


# ---- many tiles per CTA --------------------------------------------------------------------------------------------------
def many_tiles_shape(entry, axis, sms):
    """the smallest slab of tuned short axes whose pass along `axis` (2 = Z: ceil(n0*n1 / C) tiles, 1 = Y: n0 * ceil(n2 / C))
    has at least 3 tiles per CTA the device can hold: a CTA of T * C threads leaves at most min(32, 2048 / (T * C)) resident per
    SM, so every CTA of the persistent grid (SMs x occupancy, capped at the tile count) runs three or more tiles.  Ragged last
    tiles are preferred."""
    n, prec = entry[0], entry[1]
    C = entry[2][0 if axis == 2 else 1]
    need = 3 * sms * min(32, 2048 // threads(entry, axis))
    best = None
    for a in lengths(prec):
        for b in lengths(prec):
            tiles = -(-(a * b) // C) if axis == 2 else a * -(-b // C)
            if tiles < need:
                continue
            ragged = (a * b if axis == 2 else b) % C != 0
            key = (a * b, not ragged)
            if best is None or key < best[0]:
                best = (key, a, b, tiles)
    _, a, b, tiles = best
    return ((a, b, n) if axis == 2 else (a, n, b)), tiles, need


MANY = [(e, axis) for e in ENTRIES for axis in (2, 1)]


@pytest.mark.parametrize("entry,axis", MANY, ids=["%s-%s" % (entry_id(e), PASS[a][0]) for e, a in MANY])
def test_many_tiles_per_cta(entry, axis, sms):
    import scipy.fft
    prec = entry[1]
    shape, tiles, need = many_tiles_shape(entry, axis, sms)
    assert tiles >= need
    npdt = CDT[prec][0]
    ntot = int(np.prod(shape))
    assert 4 * ntot * npdt().itemsize < 2.2e9, shape   # input, output, the plan's two slabs
    rng = np.random.default_rng(entry[0] * 10 + axis)
    rdt = np.float64 if prec == DOUBLE else np.float32
    x = (rng.standard_normal(shape, dtype=rdt) + 1j * rng.standard_normal(shape, dtype=rdt)).astype(npdt)
    for direction in (FWD, BWD):
        if direction == FWD:
            dev_in = x.reshape(-1)
            ref = scipy.fft.fftn(x.astype(np.complex128), workers=-1).transpose(1, 2, 0).reshape(-1)
        else:
            dev_in = np.ascontiguousarray(x.transpose(1, 2, 0)).reshape(-1)
            ref = scipy.fft.ifftn(x.astype(np.complex128), norm="forward", workers=-1).reshape(-1)
        got, mask, fused = run_fenced(shape, prec, direction, dev_in, flags=REF_FLAGS, repeat=2)
        assert mask == 0 and not fused
        r = ratios64(got, ref, EPS[prec], ntot)
        label = "many-tile %s %s %s %s: %d tiles, >= %d per CTA" % (entry_id(entry), PASS[axis][0], "fwd" if direction == FWD else "bwd", xs(shape), tiles, tiles // (need // 3))
        print("TILE-RATIO %-52s rel_l2 %6.3f  linf %6.3f" % (label, r[0], r[1]))
        _note("many-tile", prec, r)
        assert r[0] <= ldfft.REL_L2_K and r[1] <= ldfft.LINF_K, (label, r)
        del ref, got


# ---- fused register-staged t0: bit for bit the two sweeps ------------------------------------------------------------------
@pytest.mark.parametrize("entry", ENTRIES, ids=[entry_id(e) for e in ENTRIES])
def test_fused2_is_bitwise_the_two_sweeps(entry):
    n, prec = entry[0], entry[1]
    shape = (3, n, n)
    npdt = CDT[prec][0]
    rdt = np.float64 if prec == DOUBLE else np.float32
    rng = np.random.default_rng(n)
    x = (rng.standard_normal(3 * n * n, dtype=rdt) + 1j * rng.standard_normal(3 * n * n, dtype=rdt)).astype(npdt)
    for direction, scale, kind in ((FWD, 0, "ZY"), (BWD, dfft.SCALE_BACKWARD, "YZ")):
        fi, si = {}, {}
        f, fmask, ffused = run_fenced(shape, prec, direction, x, flags=dfft.FORCE_FUSE | dfft.NO_TMA | scale, repeat=2, info=fi)
        s, smask, sfused = run_fenced(shape, prec, direction, x, flags=REF_FLAGS | scale, repeat=1, info=si)
        # an entry without this kind (roles too large for shared memory together) keeps the two sweeps under FORCE_FUSE
        has = kind not in NOT_FUSED.get((n, prec), set())
        assert ffused == has and fi["launches"] == (2 if has else 3) and fmask == 0, (ffused, fi, fmask)
        assert not sfused and si["launches"] == 3 and smask == 0, (sfused, si, smask)
        assert np.array_equal(bits(f), bits(s)), ("fused t0 differs from the two sweeps", entry_id(entry), "fwd" if direction == FWD else "bwd")


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["f64", "f32"])
def test_fused2_against_long_double(prec):
    shape = (3, 64, 64)
    for direction, scale in ((FWD, 0), (BWD, dfft.SCALE_BACKWARD)):
        dev_in, want = layouts(shape, 64, prec, direction, scale=bool(scale))
        info = {}
        got, mask, fused = run_fenced(shape, prec, direction, dev_in, flags=dfft.FORCE_FUSE | dfft.NO_TMA | scale, info=info)
        assert fused and info["launches"] == 2 and mask == 0
        check("fused2", got, want, prec, dev_in.size, "64%s %s %s" % (PN[prec], "ZY fwd" if direction == FWD else "YZ bwd scaled", xs(shape)))


# ---- generic kernel ------------------------------------------------------------------------------------------------------
GENERIC_LENGTHS = [2, 3, 5, 7, 11, 13, 121, 169, 143, 1331, 2197, 1001, 3000]
GENERIC = [(n, p) for p in (DOUBLE, FLOAT) for n in GENERIC_LENGTHS] + [(6400, DOUBLE), (12800, FLOAT)]   # + the shared-memory limits
GENERIC_CASES = [(n, p, axis) for n, p in GENERIC for axis in (2, 1, 0)]


@pytest.mark.parametrize("n,prec,axis", GENERIC_CASES, ids=["%d%s-%s" % (n, PN[p], PASS[a][0][0]) for n, p, a in GENERIC_CASES])
def test_generic_kernel_against_long_double(n, prec, axis):
    assert dfft.length_kind(n, prec) == 1
    run_axis(n, prec, axis, family="generic")


FORCED = [(n, p, axis) for p in (DOUBLE, FLOAT) for n in (4, 512, 768, 1000) for axis in (2, 1, 0)]


@pytest.mark.parametrize("n,prec,axis", FORCED, ids=["%d%s-%s" % (n, PN[p], PASS[a][0][0]) for n, p, a in FORCED])
def test_forced_generic_kernel_on_tuned_lengths(n, prec, axis, monkeypatch):
    monkeypatch.setenv("DFFT_GENERIC", "1")     # read when a plan looks up its lengths
    assert dfft.length_kind(n, prec) == 1
    run_axis(n, prec, axis, family="generic")


# ---- lines engine: four-step long lines, 2-D plans ---------------------------------------------------------------------------
# the lengths of test_gpu_parity.py::test_four_step_long_lines; in fp32, 6561, 8192 and 12000 still fit one shared-memory line
# and run as a single generic pass
FOUR_STEP = [8192, 16384, 131072, 6561, 19683, 78125, 16807, 12000]


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["f64", "f32"])
@pytest.mark.parametrize("n", FOUR_STEP)
def test_long_lines_against_long_double(n, prec):
    lines = 3
    four_step = dfft.length_kind(n, prec) == 0
    for direction in (FWD, BWD):
        ops = dfft.lines_ops(n, 1, lines, lines, n, 0, direction, prec)
        if four_step:
            assert [o["op"] for o in ops] == ["XF_TW", "Y"] and ops[0]["tw_n"] == n and ops[0]["N"] * ops[1]["N"] == n, ops
        else:
            assert dfft.length_kind(n, prec) == 1 and [(o["op"], o["N"], o["tw_n"]) for o in ops] == [("Z", n, 0)], ops
    split = "%d x %d" % (ops[0]["N"], ops[1]["N"]) if four_step else "one pass"
    rng = np.random.default_rng(n)
    x = (rng.standard_normal((lines, n)) + 1j * rng.standard_normal((lines, n))).astype(CDT[prec][0])
    plan = dfft.LinesPlan(n, 1, lines, lines, n, 0, prec)
    try:
        for direction in (FWD, BWD):
            got = run_lines(plan, x, prec, direction)
            want = ldfft.fft(x, axis=1, sign=-1 if direction == FWD else 1)
            check("four-step" if four_step else "generic", got, want, prec, n,
                  "%d%s %s %d lines (%s)" % (n, PN[prec], "fwd" if direction == FWD else "bwd", lines, split))
    finally:
        plan.destroy()


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["f64", "f32"])
def test_lines_plan_2d_against_long_double(prec):
    nx, ny, batch = 1000, 49, 3
    rng = np.random.default_rng(nx + ny)
    x = (rng.standard_normal((batch, ny, nx)) + 1j * rng.standard_normal((batch, ny, nx))).astype(CDT[prec][0])
    plan = dfft.LinesPlan(two_d=(nx, ny, batch), precision=prec)
    try:
        for direction in (FWD, BWD):
            sign = -1 if direction == FWD else 1
            got = run_lines(plan, x, prec, direction)
            want = ldfft.fft(ldfft.fft(x, axis=2, sign=sign), axis=1, sign=sign)
            check("lines-2d", got, want, prec, nx * ny, "%s%s %s %dx%dx%d" % ("2-D ", PN[prec], "fwd" if direction == FWD else "bwd", batch, ny, nx))
    finally:
        plan.destroy()


def test_zz_report_worst_ratios():
    for (family, prec), (rl2, linf) in sorted(WORST.items()):
        print("TILE-WORST %-12s %s rel_l2 %.3f linf %.3f" % (family, PN[prec], rl2, linf))
