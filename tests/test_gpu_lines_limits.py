"""The 1-D lines plans at the limits they accept, against long double (tests/ldfft.py) with the bounds of DESIGN §4: rel_l2 <= 1.0 *
eps * log2(n) and max error / rms(ref) <= 4 * eps * log2(n) (the convolve plan: twice both, for its two transforms).

- General column layouts: every tuned length in both precisions and the generic lengths of test_gpu_tile_matrix.py, as columns of
  two matrices with padded rows, a gap between the matrices, and interleaved matrices, forward and backward.  Each result is
  bit-identical to the same columns in the dense layout (the same kernel and schedule, only the strides differ), the dense one is
  held to the bounds, and every element between the columns must come back bit for bit (ld_harness.run_lines).
- Four-step long lines at the top of the range: 6400^2 fp64 and 12800^2 fp32 (the largest lengths that split into two lines of one
  shared-memory line each), 4096^2, prime powers split into two generic factors, and mixed lengths; each split asserted from the
  plan's records, enough lines for three or more tiles per resident CTA in both passes, fp32 at an odd complex64 offset.  Up to
  2^20 points the last line is checked against long double, and every line against scipy's fp64 FFT (ld_harness.ratios64).
- Buffers past 2^31 elements (fp32): contiguous lines, strided columns, four-step lines, R2C and C2R lines, the 1-D convolve plan,
  a batched 3-D plan on the plane kernel, and 2^31 - 1 rows of two points.  The whole output is checked on the device (no NaN,
  canaries intact, and each line's energy: Parseval); sampled lines -- the first, those around element 2^31, tile boundaries and
  the last -- are bit-identical to a small plan over the same data and held to the bounds.  A case is skipped, saying so, when
  the device has too little free memory; each frees its buffers before the next.

Every checked case prints a "LIMITS-RATIO" line, test_zz_report_worst_ratios the worst per family ("LIMITS-WORST"), and each case
past 2^31 the free memory it found ("LIMITS-MEM")."""
import faulthandler
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from ld_harness import CANARY, CDT, EPS, bits, ratios64, run_lines  # noqa: E402
from test_gpu_lines_conv1d import ld_conv1, run as run_conv1d  # noqa: E402
from test_gpu_real_lines import ld_irfft, ld_rfft, run as run_real  # noqa: E402
from test_gpu_tile_matrix import GENERIC_LENGTHS  # noqa: E402
from test_lines_layouts_dry_run import line_offsets  # noqa: E402
from tile_entries import BY, DOUBLE, FLOAT, lengths  # noqa: E402

FWD, BWD = dfft.FORWARD, dfft.BACKWARD
PN = {DOUBLE: "f64", FLOAT: "f32"}
GiB = 1 << 30
LIMIT = 1 << 31
WORST = {}


@pytest.fixture(autouse=True)
def _watchdog(monkeypatch):
    # a host-side hang inside libdfft.so cannot be interrupted by a Python-level signal handler; the cases past 2^31 elements fill,
    # transform and scan tens of GB
    faulthandler.dump_traceback_later(600, exit=True, file=sys.stderr)
    for var in ("DFFT_GENERIC", "DFFT_VARIANT", "DFFT_NO_LONG_LINES", "DFFT_NO_PLANE", "DFFT_FORCE_PLANE"):
        monkeypatch.delenv(var, raising=False)
    yield
    faulthandler.cancel_dump_traceback_later()


@pytest.fixture(scope="module", autouse=True)
def _long_double():
    assert np.finfo(np.longdouble).eps <= ldfft.LD_EPS_MAX, "np.longdouble is not wider than double: no reference for the fp64 bounds"


def check(family, got, want, prec, ntot, label, k=1, big=False):
    """both ratios against the reference (long double, or with big=True scipy's fp64 through ratios64), bounds times k"""
    r = ratios64(got, want, EPS[prec], ntot) if big else ldfft.ratios(got, want, EPS[prec], ntot)
    print("LIMITS-RATIO %-12s %-56s rel_l2 %6.3f  linf %6.3f" % (family, label, r[0], r[1]))
    w = WORST.get((family, prec), (0.0, 0.0))
    WORST[family, prec] = (max(w[0], r[0]), max(w[1], r[1]))
    assert r[0] <= k * ldfft.REL_L2_K and r[1] <= k * ldfft.LINF_K, (label, r)


def same_bits(a, b, what):
    assert a.shape == b.shape and np.array_equal(bits(a), bits(b)), what


def random_lines(shape, prec, seed):
    rng = np.random.default_rng(seed)
    rdt = np.float64 if prec == DOUBLE else np.float32
    return (rng.standard_normal(shape, dtype=rdt) + 1j * rng.standard_normal(shape, dtype=rdt)).astype(CDT[prec][0])


# ---- general column layouts ----------------------------------------------------------------------------------------------
INNER, MATS = 9, 2   # 9 columns: a ragged last tile for every column tile width (2 .. 32, generic 1 .. 8)
LAYOUT_CASES = [(n, p) for p in (DOUBLE, FLOAT) for n in lengths(p)] + [(n, p) for p in (DOUBLE, FLOAT) for n in GENERIC_LENGTHS]


def column_layouts(n):
    """{name: (stride, outer_dist)} of MATS matrices of n rows and INNER columns"""
    return {"dense": (INNER, n * INNER), "padded": (INNER + 3, n * (INNER + 3)), "gapped": (INNER, n * INNER + 7),
            "interleaved": (MATS * INNER, INNER)}


@pytest.mark.parametrize("n,prec", LAYOUT_CASES, ids=["%d%s" % (n, PN[p]) for n, p in LAYOUT_CASES])
def test_column_layouts(n, prec):
    nlines = INNER * MATS
    x = random_lines((nlines, n), prec, n)
    got = {}
    for name, (stride, outer) in column_layouts(n).items():
        ops = dfft.lines_ops(n, stride, nlines, INNER, 1, outer, FWD, prec)
        assert [(o["op"], o["ia"]) for o in ops] == [("Y", [outer, ops[0]["C"], 1, stride])] and INNER % ops[0]["C"], ops
        off = line_offsets(n, stride, nlines, INNER, 1, outer)
        plan = dfft.LinesPlan(n, stride, nlines, INNER, 1, outer, prec)
        try:
            for direction in (FWD, BWD):
                got[name, direction] = run_lines(plan, x, prec, direction, offsets=off, size=int(off.max()) + 1)
        finally:
            plan.destroy()
    for direction in (FWD, BWD):
        dense = got["dense", direction]
        d = "fwd" if direction == FWD else "bwd"
        for name in column_layouts(n):
            same_bits(got[name, direction], dense, (name, d))
        check("layouts", dense, ldfft.fft(x, axis=1, sign=-1 if direction == FWD else 1), prec, n,
              "%d%s %s %d columns x %d matrices" % (n, PN[prec], d, INNER, MATS))


# ---- four-step long lines at the top of the range -------------------------------------------------------------------------
# (n, precision, split n1 x n2)
FOUR_STEP = ([(6400 * 6400, DOUBLE, (6400, 6400)), (4096 * 4096, DOUBLE, (4096, 4096)),
              (12800 * 12800, FLOAT, (12800, 12800)), (1 << 24, FLOAT, (4096, 4096))]
             + [(p ** k, prec, (p ** (k // 2),) * 2) for p, k in ((3, 14), (5, 10), (7, 8), (11, 6), (13, 6)) for prec in (DOUBLE, FLOAT)]
             + [(n, prec, s) for n, s in ((1 << 20, (1024, 1024)), (10 ** 6, (1000, 1000)), (768 * 1024, (768, 1024))) for prec in (DOUBLE, FLOAT)])


def resident_bound(N, C, prec, axis):
    """at most this many CTAs of a pass over lines of N points sit on one SM: min(32, 2048 / threads), threads = N / R * C for a
    tuned entry (R of its X (axis 0) or Y (axis 1) schedule), 256 for the run-time-scheduled kernel"""
    if dfft.length_kind(N, prec) == 2:
        e = BY[N, prec]
        assert e[2][2 if axis == 0 else 1] == C, (N, C, e)
        threads = N // e[3][2 if axis == 0 else 1] * C
    else:
        threads = 256
    return min(32, 2048 // threads)


@pytest.mark.parametrize("n,prec,split", FOUR_STEP, ids=["%d%s" % (n, PN[p]) for n, p, _ in FOUR_STEP])
def test_four_step_at_the_top_of_the_range(n, prec, split):
    import scipy.fft
    assert dfft.length_kind(n, prec) == 0
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ops = dfft.lines_ops(n, 1, 1, 1, n, 0, FWD, prec)
    assert [o["op"] for o in ops] == ["XF_TW", "Y"] and (ops[0]["N"], ops[1]["N"]) == split and ops[0]["tw_n"] == n, ops
    # enough lines that every CTA of both persistent grids runs three or more tiles
    need = [3 * sms * resident_bound(o["N"], o["C"], prec, axis) for o, axis in zip(ops, (0, 1))]
    nlines = max([1] + [-(-k // o["ntiles"]) for k, o in zip(need, ops)])
    for direction in (FWD, BWD):
        ops = dfft.lines_ops(n, 1, nlines, nlines, n, 0, direction, prec)
        assert [o["op"] for o in ops] == ["XF_TW", "Y"] and all(o["ntiles"] >= k for o, k in zip(ops, need)), (ops, need)
    offset = 1 if prec == FLOAT else 0
    x = random_lines((nlines, n), prec, n % 1000003)
    plan = dfft.LinesPlan(n, 1, nlines, nlines, n, 0, prec)
    try:
        for direction in (FWD, BWD):
            d = "fwd" if direction == FWD else "bwd"
            label = "%d%s %s %d x %d, %d lines%s" % (n, PN[prec], d, split[0], split[1], nlines, " offset 1" if offset else "")
            got = run_lines(plan, x, prec, direction, offset=offset)
            sign = -1 if direction == FWD else 1
            if n <= 1 << 20:
                check("four-step", got[-1], ldfft.fft(x[-1], sign=sign), prec, n, label + " last line, long double")
            ref = scipy.fft.fft(x.astype(np.complex128), axis=1, workers=-1) if sign < 0 else \
                scipy.fft.ifft(x.astype(np.complex128), axis=1, norm="forward", workers=-1)
            check("four-step", got, ref, prec, n, label + ", scipy fp64", big=True)
            del got, ref
    finally:
        plan.destroy()


# ---- buffers past 2^31 elements ------------------------------------------------------------------------------------------
def free_or_skip(need, what):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    print("LIMITS-MEM %-40s needs %5.1f GiB; %5.1f of %5.1f GiB free" % (what, need / GiB, free / GiB, total / GiB))
    if free < need + 2 * GiB:
        pytest.skip("%s needs %.1f GiB of device memory; %.1f GiB are free" % (what, need / GiB, free / GiB))


def release():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def arena(count, tdt, seed):
    """(arena, view, fence): CANARY random elements, `count` random elements in `view`, CANARY random elements"""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    a = torch.empty(count + 2 * CANARY, dtype=tdt, device="cuda")
    view = a[CANARY: CANARY + count]
    for chunk in a.split(1 << 28):
        (torch.view_as_real(chunk) if chunk.is_complex() else chunk).normal_(generator=g)
    fence = torch.cat([a[:CANARY], a[CANARY + count:]]).clone()
    return a, view, fence


def intact(a, fence, view, what):
    """no NaN in `view`, and the canaries of its arena unchanged"""
    for chunk in view.split(1 << 27):
        assert not torch.isnan(torch.view_as_real(chunk) if chunk.is_complex() else chunk).any().item(), "NaN in the output of " + what
    assert torch.equal(torch.cat([a[:CANARY], a[-CANARY:]]), fence), "canary overwritten: " + what


def energies(rows, weights=None, chunk=1 << 14):
    """sum of |.|^2 over the last axis of each row (weights: per element of the last axis), in fp64"""
    out = []
    for c in rows.split(chunk):
        sq = (torch.view_as_real(c).double() ** 2).sum(-1) if c.is_complex() else c.double() ** 2
        out.append((sq if weights is None else sq * weights).sum(-1))
    return torch.cat(out)


def parseval(after, before, factor, what, rtol=1e-4):
    """every line (column, volume) holds factor times its input's energy: a line that was skipped, transformed twice or mixed
    with another is off by a factor of the order of n"""
    dev = (after / (factor * before) - 1).abs()
    worst = dev.max().item()
    print("LIMITS-PARSEVAL %-40s %d lines, worst relative deviation %.2e" % (what, before.numel(), worst))
    assert worst <= rtol, (what, worst, int(dev.argmax().item()))


def samples(count, per, C):
    """line indices to check: the first, tile boundaries, those around element 2^31 (lines of `per` elements) and the last"""
    at = LIMIT // per
    t = at // C * C
    s = {0, 1, C - 1, C, t - 1, t, at - 1, at, at + 1, count - C - 1, count - C, count - 2, count - 1}
    return np.array(sorted(i for i in s if 0 <= i < count))


def test_contiguous_lines_past_2_31_elements():
    n, nl = 1024, (1 << 21) + 5
    assert n * nl > LIMIT
    free_or_skip(n * nl * 8, "contiguous C2C 1024 x (2^21 + 5) f32")
    ops = dfft.lines_ops(n, 1, nl, nl, n, 0, FWD, FLOAT)
    assert [(o["op"], o["W"]) for o in ops] == [("Z", nl)], ops
    idx = samples(nl, n, ops[0]["C"])
    a, view, fence = arena(n * nl, torch.complex64, 1)
    try:
        lines = view.view(nl, n)
        x, e0 = lines[idx].cpu().numpy(), energies(lines)
        plan = dfft.LinesPlan(n, 1, nl, nl, n, 0, FLOAT)
        try:
            torch.cuda.synchronize()
            plan.execute(view.data_ptr(), FWD)
            plan.synchronize()
        finally:
            plan.destroy()
        got = lines[idx].cpu().numpy()
        intact(a, fence, view, "contiguous lines")
        parseval(energies(lines), e0, n, "contiguous C2C")
    finally:
        del a, view, fence
        release()
    small = dfft.LinesPlan(n, 1, len(idx), len(idx), n, 0, FLOAT)
    try:
        same_bits(got, run_lines(small, x, FLOAT, FWD, repeat=1), "contiguous lines against a small plan")
    finally:
        small.destroy()
    check("past-2^31", got, ldfft.fft(x, axis=1), FLOAT, n, "C2C 1024f32 %d sampled lines of %d" % (len(idx), nl))


def test_strided_columns_spanning_past_2_31_elements():
    n, cols = 1024, (1 << 21) + 3
    assert n * cols > LIMIT
    free_or_skip(n * cols * 8, "strided 1024 rows x (2^21 + 3) columns f32")
    ops = dfft.lines_ops(n, cols, cols, cols, 1, 0, FWD, FLOAT)
    assert [(o["op"], o["W"]) for o in ops] == [("Y", cols)], ops
    C = ops[0]["C"]
    cross = LIMIT - (n - 1) * cols     # the column whose last point is element 2^31
    idx = np.array(sorted({0, 1, C - 1, C, cross - 1, cross, cross // C * C, cols - 2, cols - 1}))
    a, view, fence = arena(n * cols, torch.complex64, 2)
    try:
        mat = view.view(n, cols)
        x = mat[:, idx].T.contiguous().cpu().numpy()
        e0 = torch.zeros(cols, dtype=torch.float64, device="cuda")
        for rows in mat.split(16):
            e0 += (torch.view_as_real(rows).double() ** 2).sum((0, 2))
        plan = dfft.LinesPlan(n, cols, cols, cols, 1, 0, FLOAT)
        try:
            torch.cuda.synchronize()
            plan.execute(view.data_ptr(), FWD)
            plan.synchronize()
        finally:
            plan.destroy()
        got = mat[:, idx].T.contiguous().cpu().numpy()
        intact(a, fence, view, "strided columns")
        e1 = torch.zeros_like(e0)
        for rows in mat.split(16):
            e1 += (torch.view_as_real(rows).double() ** 2).sum((0, 2))
        parseval(e1, e0, n, "strided columns")
    finally:
        del a, view, fence
        release()
    k = len(idx)
    small = dfft.LinesPlan(n, k, k, k, 1, 0, FLOAT)
    try:
        off = line_offsets(n, k, k, k, 1, 0)
        same_bits(got, run_lines(small, x, FLOAT, FWD, repeat=1, offsets=off, size=n * k), "strided columns against a small plan")
    finally:
        small.destroy()
    check("past-2^31", got, ldfft.fft(x, axis=1), FLOAT, n, "columns 1024f32 %d sampled of %d" % (k, cols))


def test_four_step_lines_past_2_31_elements():
    import scipy.fft
    n, nl = 1 << 24, 129
    assert n * nl > LIMIT
    free_or_skip(2 * n * nl * 8, "four-step 2^24 x 129 f32 + temporary")
    ops = dfft.lines_ops(n, 1, nl, nl, n, 0, FWD, FLOAT)
    assert [(o["op"], o["N"]) for o in ops] == [("XF_TW", 4096), ("Y", 4096)], ops
    idx = np.array([0, 1, nl - 2, nl - 1])   # line 128 starts at element 2^31
    a, view, fence = arena(n * nl, torch.complex64, 3)
    try:
        lines = view.view(nl, n)
        x, e0 = lines[idx].cpu().numpy(), energies(lines, chunk=1)
        plan = dfft.LinesPlan(n, 1, nl, nl, n, 0, FLOAT)
        try:
            torch.cuda.synchronize()
            plan.execute(view.data_ptr(), FWD)
            plan.synchronize()
        finally:
            plan.destroy()
        got = lines[idx].cpu().numpy()
        intact(a, fence, view, "four-step lines")
        parseval(energies(lines, chunk=1), e0, n, "four-step")
    finally:
        del a, view, fence
        release()
    small = dfft.LinesPlan(n, 1, len(idx), len(idx), n, 0, FLOAT)
    try:
        same_bits(got, run_lines(small, x, FLOAT, FWD, repeat=1), "four-step lines against a small plan")
    finally:
        small.destroy()
    ref = scipy.fft.fft(x.astype(np.complex128), axis=1, workers=-1)
    check("past-2^31", got, ref, FLOAT, n, "four-step 2^24f32 lines %s of %d, scipy fp64" % (idx.tolist(), nl), big=True)


def test_real_lines_past_2_31_elements():
    n, nl = 1024, (1 << 21) + 6
    H = n // 2 + 1
    assert n * nl > LIMIT
    free_or_skip(n * nl * 4 + H * nl * 8, "R2C / C2R 1024 x (2^21 + 6) f32")
    at = LIMIT // n
    idx = np.array(sorted({p + i for p in (0, 2, at - 2, at, nl - 2) for i in (0, 1)}))   # even-aligned pairs
    w = torch.full((H,), 2.0, dtype=torch.float64, device="cuda")
    w[0] = w[-1] = 1
    r, rv, rfence = arena(n * nl, torch.float32, 4)
    c, cv, cfence = arena(H * nl, torch.complex64, 5)
    try:
        real, spec = rv.view(nl, n), cv.view(nl, H)
        x, e0 = real[idx].cpu().numpy(), energies(real)
        cv.fill_(complex(float("nan"), float("nan")))
        plan = dfft.RealLinesPlan(n, nl, FLOAT)
        try:
            torch.cuda.synchronize()
            plan.execute(rv.data_ptr(), cv.data_ptr(), FWD)
            plan.synchronize()
            S = spec[idx].cpu().numpy()
            intact(c, cfence, cv, "R2C")
            es = energies(spec, w)
            parseval(es, e0, n, "R2C")
            assert torch.equal(energies(real), e0), "R2C changed its input"
            rv.fill_(float("nan"))
            torch.cuda.synchronize()
            plan.execute(cv.data_ptr(), rv.data_ptr(), BWD)
            plan.synchronize()
        finally:
            plan.destroy()
        y = real[idx].cpu().numpy()
        intact(r, rfence, rv, "C2R")
        assert torch.equal(energies(spec, w), es), "C2R changed its input"
        parseval(energies(real), e0, n * n, "C2R of the R2C")
    finally:
        del r, rv, c, cv, real, spec
        release()
    k = len(idx)
    same_bits(S, run_real(FWD, x.reshape(-1), FLOAT, n, k, repeat=1).reshape(k, H), "R2C against a small plan")
    same_bits(y, run_real(BWD, S.reshape(-1), FLOAT, n, k, repeat=1).reshape(k, n), "C2R against a small plan")
    check("past-2^31", S, ld_rfft(x, (-1,)), FLOAT, n, "R2C 1024f32 %d sampled lines of %d" % (k, nl))
    check("past-2^31", y, ld_irfft(S, n), FLOAT, n, "C2R 1024f32 %d sampled lines of %d" % (k, nl))


def test_convolve_1d_past_2_31_elements():
    n, nl = 1024, (1 << 21) + 5
    assert n * nl > LIMIT
    free_or_skip(n * nl * 8, "convolve 1-D 1024 x (2^21 + 5) f32")
    ops = dfft.lines_conv_1d_ops(n, nl, FLOAT)
    assert len(ops) == 1 and ops[0]["W"] == nl, ops
    idx = samples(nl, n, ops[0]["C"])
    rng = np.random.default_rng(6)
    m = np.exp(2j * np.pi * rng.uniform(size=n)).astype(np.complex64)   # |m| = 1: each line keeps n^2 times its energy
    a, view, fence = arena(n * nl, torch.complex64, 6)
    try:
        lines = view.view(nl, n)
        mult = torch.from_numpy(m).cuda()
        x, e0 = lines[idx].cpu().numpy(), energies(lines)
        plan = dfft.LinesConvolvePlan(one_d=(n, nl), precision=FLOAT)
        try:
            torch.cuda.synchronize()
            plan.execute(view.data_ptr(), view.data_ptr(), mult.data_ptr(), 1)
            plan.synchronize()
        finally:
            plan.destroy()
        got = lines[idx].cpu().numpy()
        intact(a, fence, view, "convolve 1-D")
        parseval(energies(lines), e0, n * n, "convolve 1-D")
    finally:
        del a, view, fence
        release()
    same_bits(got, run_conv1d(n, len(idx), FLOAT, x, m, repeat=1), "convolve 1-D against a small plan")
    check("past-2^31", got, ld_conv1(x, m, False), FLOAT, n, "convolve 1024f32 %d sampled lines of %d" % (len(idx), nl), k=2)


def test_batched_3d_on_the_plane_kernel_past_2_31_elements():
    nx, ny, nz, batch = 64, 64, 48, 10924
    V = nx * ny * nz
    assert V * batch > LIMIT and V * (batch - 2) < LIMIT < V * (batch - 1)   # volume batch - 2 holds element 2^31
    free_or_skip(V * batch * 8, "3-D 64x64x48 x 10924 f32")
    assert [o["op"] for o in dfft.lines_3d_ops(nx, ny, nz, batch, FWD, FLOAT)] == ["XY_PLANE", "Y"]
    idx = np.array([0, 1, batch - 3, batch - 2, batch - 1])
    a, view, fence = arena(V * batch, torch.complex64, 7)
    try:
        vols = view.view(batch, V)
        x, e0 = vols[idx].cpu().numpy().reshape(-1, nz, ny, nx), energies(vols, chunk=64)
        plan = dfft.LinesPlan(three_d=(nx, ny, nz, batch), precision=FLOAT)
        try:
            torch.cuda.synchronize()
            plan.execute(view.data_ptr(), FWD)
            plan.synchronize()
        finally:
            plan.destroy()
        got = vols[idx].cpu().numpy().reshape(x.shape)
        intact(a, fence, view, "3-D")
        parseval(energies(vols, chunk=64), e0, V, "3-D volumes")
    finally:
        del a, view, fence
        release()
    small = dfft.LinesPlan(three_d=(nx, ny, nz, len(idx)), precision=FLOAT)
    try:
        same_bits(got, run_lines(small, x, FLOAT, FWD, repeat=1), "3-D volumes against a small plan")
    finally:
        small.destroy()
    ld = [0, 3]    # the first volume and the one that holds element 2^31
    want = x[ld]
    for ax in (3, 2, 1):
        want = ldfft.fft(want, axis=ax)
    check("past-2^31", got[ld], want, FLOAT, V, "3-D 64x64x48f32 volumes %s of %d" % (idx[ld].tolist(), batch))


def test_2_31_minus_1_rows():
    """the row limit itself: 2^31 - 1 lines of two points, 32 GiB in place.  The input is small integers that depend on the line
    index, so every line's transform is known exactly and the whole output is compared on the device"""
    n, nl = 2, LIMIT - 1
    free_or_skip(n * nl * 8, "2^31 - 1 rows of 2 points f32")
    ops = dfft.lines_ops(n, 1, nl, nl, n, 0, FWD, FLOAT)
    assert [(o["op"], o["W"]) for o in ops] == [("Z", nl)], ops
    idx = samples(nl, n, ops[0]["C"])
    a = torch.empty(n * nl + 2 * CANARY, dtype=torch.complex64, device="cuda")
    try:
        view = a[CANARY: CANARY + n * nl]
        fence = torch.randn(2 * CANARY, dtype=torch.complex64, device="cuda")
        a[:CANARY], a[-CANARY:] = fence[:CANARY], fence[CANARY:]
        pts = torch.view_as_real(view.view(nl, n))          # [line][point][re, im]
        step = 1 << 26

        def structured(s, e):
            l = torch.arange(s, e, device="cuda", dtype=torch.int64)
            return [(l % p).float() for p in (4093, 4091, 509, 503)]

        for s in range(0, nl, step):
            a0, b0, c0, d0 = structured(s, min(s + step, nl))
            pts[s: s + step, 0, 0], pts[s: s + step, 0, 1], pts[s: s + step, 1, 0], pts[s: s + step, 1, 1] = a0, b0, c0, d0
        x = view.view(nl, n)[idx].cpu().numpy()
        plan = dfft.LinesPlan(n, 1, nl, nl, n, 0, FLOAT)
        try:
            torch.cuda.synchronize()
            plan.execute(view.data_ptr(), FWD)
            plan.synchronize()
        finally:
            plan.destroy()
        got = view.view(nl, n)[idx].cpu().numpy()
        assert torch.equal(torch.cat([a[:CANARY], a[-CANARY:]]), fence), "canary overwritten"
        for s in range(0, nl, step):
            a0, b0, c0, d0 = structured(s, min(s + step, nl))
            want = torch.stack([torch.stack([a0 + c0, b0 + d0], -1), torch.stack([a0 - c0, b0 - d0], -1)], 1)
            assert torch.equal(pts[s: s + step], want), "lines %d .. %d differ from their exact transforms" % (s, min(s + step, nl) - 1)
        print("LIMITS-EXACT 2^31 - 1 rows of 2 points: every line equals its exact transform")
    finally:
        del a
        release()
    small = dfft.LinesPlan(n, 1, len(idx), len(idx), n, 0, FLOAT)
    try:
        same_bits(got, run_lines(small, x, FLOAT, FWD, repeat=1), "2^31 - 1 rows against a small plan")
    finally:
        small.destroy()
    check("past-2^31", got, ldfft.fft(x, axis=1), FLOAT, n, "2 points f32 %d sampled lines of %d" % (len(idx), nl))


def test_zz_report_worst_ratios():
    for (family, prec), (rl2, linf) in sorted(WORST.items()):
        print("LIMITS-WORST %-12s %s rel_l2 %.3f linf %.3f" % (family, PN[prec], rl2, linf))
