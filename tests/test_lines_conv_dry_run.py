"""CPU tests of the batched 3-D convolve lines plans (dfft_lines_plan_create_convolve_3d / _r2c_3d) without a GPU.

dfft_debug_lines_conv_3d_ops records the passes one execute launches.  They are interpreted with the existing interpreters
(run_pass for the C2C passes, run_real for the real passes, run_plane for the plane kernel) plus run_xconv below for the
column pass that transforms along z, multiplies and transforms back.  The result is compared with numpy's
ifftn(fftn(a) * m) * N and irfftn(rfftn(a) * m) * N over axes (1, 2, 3), for a multiplier shared by every volume and one per
volume, scaled and unscaled, in place and out of place.  Every buffer starts NaN-filled with canaries past its end, so a read
outside a buffer, a missed store or a write past an end shows up; `in` (when distinct) and the multiplier must come back
unchanged.  The kernels' arithmetic is checked on the GPU by test_gpu_lines_conv.py."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_dry_run import IN, MID, OUT, decode, run_pass
from test_lines3d_dry_run import run_plane
from test_r2c_dry_run import run_real
from test_real_lines_dry_run import CANARY, PAD, bufid

TEMP = MID
MULT = 8
PLANE_LENGTHS = (16, 32, 64)


def run_xconv(m, op):
    """XCONV: per column, numpy's FFT, the product with the multiplier at the same position (without the tile coordinate a's
    a * SA when "shared"), the inverse (unnormalised), the optional scale; stored through the output map"""
    N, C, G, W = op["N"], op["C"], op["G"], op["W"]
    SAi, SBi, csi, esi = op["ia"]
    SAo, SBo, cso, eso = op["oa"]
    e = np.arange(N)
    src, soff = m.view(op["in"])
    mul, moff = m.view(op["mult"])
    staged = []
    for tile in range(op["ntiles"]):
        a, b = divmod(tile, G)
        for c in range(C):
            if b * C + c >= W:
                continue
            rel = b * SBi + c * csi + e * esi
            mrel = rel if op["shared"] else a * SAi + rel
            x = np.fft.ifft(np.fft.fft(src[soff + a * SAi + rel]) * mul[moff + mrel]) * N
            if op["do_scale"]:
                x = x * op["scale"]
            staged.append((a, b, c, x))
    dst, doff = m.view(op["out"])
    for a, b, c, x in staged:
        dst[doff + a * SAo + b * SBo + c * cso + e * eso] = x


class ConvMachine:
    """device 0 only: complex128 arrays of the given lengths + PAD, NaN-filled with CANARY in the pad; `in` aliases `out`
    when in place"""

    def __init__(self, sizes, inplace):
        self.mem = {}
        for b, n in sizes.items():
            arr = np.full(n + PAD, np.nan, dtype=np.complex128)
            arr[n:] = CANARY
            self.mem[b] = arr
        if inplace:
            self.mem[IN] = self.mem[OUT]

    def buf(self, dev, b):
        assert dev == 0, dev
        return self.mem[b]

    def view(self, addr):
        dev, b, off = decode(addr)
        return self.buf(dev, b), off


def ops_of(nx, ny, nz, batch, real=False, flags=0, mult_count=1, precision=dfft.DOUBLE):
    return dfft.lines_conv_3d_ops(nx, ny, nz, batch, precision, real, flags, mult_count)


def simulate(nx, ny, nz, batch, a, M, real=False, flags=0, inplace=False, precision=dfft.DOUBLE):
    """a: [batch][nz][ny][nx] input; M: the multiplier, one volume (shared) or [batch] of them"""
    H = nx // 2 + 1
    vol = nx * ny * nz
    mvol = nz * ny * (H if real else nx)
    mult_count = 1 if M.ndim == 3 else batch
    io = -(-vol * batch // 2) if real else vol * batch   # complex128 slots holding the caller's buffer
    sizes = {IN: io, OUT: io, MULT: mvol * mult_count}
    if real:
        sizes[TEMP] = nz * ny * H * batch
    m = ConvMachine(sizes, inplace)
    inb = m.mem[IN].view(np.float64) if real else m.mem[IN]
    inb[: a.size] = a.reshape(-1)
    m.mem[MULT][: M.size] = M.reshape(-1)
    keep_in, keep_mult = m.mem[IN].copy(), m.mem[MULT].copy()
    ops = ops_of(nx, ny, nz, batch, real, flags, mult_count, precision)
    for op in ops:
        assert bufid(op["out"]) not in (MULT,) and (inplace or bufid(op["out"]) != IN), ("a pass writes a read-only buffer", op["op"])
        if op["op"] == "XY_PLANE":
            run_plane(m, op)
        elif op["op"] == "XCONV":
            run_xconv(m, op)
        elif op["op"] in ("Z_R2C", "Z_C2R"):
            run_real(m, op)
        else:
            run_pass(m, op)
    assert np.array_equal(m.mem[MULT], keep_mult, equal_nan=True), "the multiplier was written"
    if not inplace:
        assert np.array_equal(m.mem[IN], keep_in, equal_nan=True), "`in` was written"
    for b, arr in m.mem.items():
        assert np.all(arr[sizes[b]:] == CANARY), f"write past the end of buffer {b}"
    out = m.mem[OUT].view(np.float64)[: vol * batch] if real else m.mem[OUT][: vol * batch]
    got = out.copy()
    assert not np.isnan(got.view(np.float64)).any(), "an output element was never written (or read NaN)"
    return got, ops


def want_c2c(a, M, scaled):
    N = np.prod(a.shape[1:])
    r = np.fft.ifftn(np.fft.fftn(a, axes=(1, 2, 3)) * M, axes=(1, 2, 3))
    return r if scaled else r * N


def want_r2c(a, M, scaled):
    N = np.prod(a.shape[1:])
    r = np.fft.irfftn(np.fft.rfftn(a, axes=(1, 2, 3)) * M, s=a.shape[1:], axes=(1, 2, 3))
    return r if scaled else r * N


def check(got, want):
    want = want.reshape(-1)
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-11 * max(1.0, np.abs(want).max())


def rand_c(rng, shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


# (nx, ny, nz, batch): the plane lengths with nz 16 / 32 / 64 and ragged batches; non-square, generic nx / ny, and mixed tuned
# lengths; odd nz (9, 125)
C2C_SHAPES = [(16, 16, 16, 3), (16, 16, 64, 2), (32, 32, 32, 2), (32, 32, 16, 5), (64, 64, 16, 1), (64, 64, 64, 1),
              (14, 22, 16, 2), (16, 8, 32, 3), (48, 48, 12, 1), (12, 24, 9, 3), (22, 14, 125, 1), (9, 9, 9, 2), (10, 6, 4, 1)]


@pytest.mark.parametrize("nx,ny,nz,batch", C2C_SHAPES)
def test_c2c_convolution_matches_numpy(nx, ny, nz, batch):
    rng = np.random.default_rng(nx * 10007 + ny * 101 + nz * 7 + batch)
    a = rand_c(rng, (batch, nz, ny, nx))
    plane = nx == ny and nx in PLANE_LENGTHS
    seq = ["XY_PLANE", "XCONV", "XY_PLANE"] if plane else ["Z", "Y", "XCONV", "Y", "Z"]
    # shared, unscaled, out of place / one per volume, scaled, in place
    M = rand_c(rng, (nz, ny, nx))
    got, ops = simulate(nx, ny, nz, batch, a, M)
    assert [o["op"] for o in ops] == seq
    assert [o["inv"] for o in ops if o["op"] != "XCONV"] == [0] * (len(seq) // 2) + [1] * (len(seq) // 2)
    assert [(bufid(o["in"]), bufid(o["out"])) for o in ops] == [(IN, OUT)] + [(OUT, OUT)] * (len(seq) - 1)
    conv = ops[len(seq) // 2]
    assert conv["N"] == nz and conv["shared"] == 1 and bufid(conv["mult"]) == MULT and not conv["do_scale"]
    check(got, want_c2c(a, M, False))
    Mb = rand_c(rng, (batch, nz, ny, nx))
    got, ops = simulate(nx, ny, nz, batch, a, Mb, flags=dfft.SCALE_BACKWARD, inplace=True)
    conv = ops[len(seq) // 2]
    assert conv["shared"] == (batch == 1) and conv["do_scale"] and conv["scale"] == pytest.approx(1.0 / (nx * ny * nz), rel=1e-15)
    check(got, want_c2c(a, Mb, True))


# tuned even / odd nx, generic nx and ny, odd nz
R2C_SHAPES = [(16, 16, 16, 3), (64, 64, 64, 1), (9, 8, 6, 3), (14, 22, 16, 2), (21, 10, 9, 1), (32, 12, 125, 1), (2, 3, 4, 2)]


@pytest.mark.parametrize("nx,ny,nz,batch", R2C_SHAPES)
def test_r2c_convolution_matches_numpy(nx, ny, nz, batch):
    rng = np.random.default_rng(nx * 1000 + ny * 10 + nz + batch)
    H = nx // 2 + 1
    a = rng.standard_normal((batch, nz, ny, nx))
    M = rand_c(rng, (nz, ny, H))   # not Hermitian: the C2R ignores what numpy's irfftn ignores
    got, ops = simulate(nx, ny, nz, batch, a, M, real=True)
    assert [o["op"] for o in ops] == ["Z_R2C", "Y", "XCONV", "Y", "Z_C2R"]
    assert [(bufid(o["in"]), bufid(o["out"])) for o in ops] == [(IN, TEMP)] + [(TEMP, TEMP)] * 3 + [(TEMP, OUT)]
    assert [o["inv"] for o in ops[1:4]] == [0, 0, 1] and ops[1]["N"] == ny and ops[2]["N"] == nz
    check(got, want_r2c(a, M, False))
    Mb = rand_c(rng, (batch, nz, ny, H))
    for inplace in (False, True):
        got, ops = simulate(nx, ny, nz, batch, a, Mb, real=True, flags=dfft.SCALE_BACKWARD, inplace=inplace)
        assert ops[2]["shared"] == (batch == 1) and ops[2]["do_scale"]   # mult_count == batch == 1 is the shared case
        check(got, want_r2c(a, Mb, True))


@pytest.mark.parametrize("n", PLANE_LENGTHS)
@pytest.mark.parametrize("precision", [dfft.DOUBLE, dfft.FLOAT])
def test_plane_selection_follows_the_3d_lines_plan(n, precision, monkeypatch):
    """the plane kernel runs exactly where dfft_lines_plan_create_3d would run it, read from the environment at creation"""
    def seq(**kw):
        return [o["op"] for o in ops_of(n, n, 16, 3, precision=precision, **kw)]
    plane3d = any(o["op"] == "XY_PLANE" for o in dfft.lines_3d_ops(n, n, 16, 3, dfft.FORWARD, precision))
    assert seq() == (["XY_PLANE", "XCONV", "XY_PLANE"] if plane3d else ["Z", "Y", "XCONV", "Y", "Z"])
    monkeypatch.setenv("DFFT_NO_PLANE", "1")
    assert seq() == ["Z", "Y", "XCONV", "Y", "Z"]
    monkeypatch.delenv("DFFT_NO_PLANE")
    monkeypatch.setenv("DFFT_FORCE_PLANE", "1")
    assert seq() == ["XY_PLANE", "XCONV", "XY_PLANE"]
    monkeypatch.delenv("DFFT_FORCE_PLANE")
    assert seq(real=True) == ["Z_R2C", "Y", "XCONV", "Y", "Z_C2R"]


@pytest.mark.parametrize("precision", [dfft.DOUBLE, dfft.FLOAT])
def test_single_precision_schedule_matches_numpy(precision):
    """fp32 entries tile differently (other C per pass); the schedule is the same arithmetic"""
    rng = np.random.default_rng(11)
    a = rand_c(rng, (3, 32, 24, 20))
    M = rand_c(rng, (32, 24, 20))
    got, _ = simulate(20, 24, 32, 3, a, M, precision=precision)
    check(got, want_c2c(a, M, False))


def code(fn, *args, **kw):
    try:
        fn(*args, **kw)
    except dfft.DfftError as e:
        return int(str(e).split("(")[1].split(")")[0])
    return 0


@pytest.mark.parametrize("real", [False, True])
def test_unsupported_requests_are_refused(real, monkeypatch):
    def c(nx, ny, nz, batch, flags=0, mult_count=1, precision=dfft.DOUBLE):
        return code(ops_of, nx, ny, nz, batch, real, flags, mult_count, precision)
    assert c(16, 16, 16, 4) == 0 and c(14, 22, 16, 1) == 0 and c(16, 16, 16, 0) == 0 and c(16, 16, 16, 4, mult_count=4) == 0
    assert c(16, 16, 16, 4, flags=dfft.SCALE_BACKWARD) == 0
    for nz in (14, 22, 26, 17):                              # no tuned kernel (generic lengths) or no kernel at all
        assert dfft.length_kind(nz, dfft.DOUBLE) != 2
        assert c(16, 16, nz, 1) == -3, nz
    assert c(17, 16, 16, 1) == -3 and c(16, 17, 16, 1) == -3
    assert c(16, 1, 16, 1) == -3                             # no strided pass of length 1
    assert c(16, 16, 16, 1 << 23) == -3 and c(16, 16, 16, (1 << 23) - 1) == 0   # 2^31 rows
    assert c(0, 16, 16, 1) in (-1, -3) and c(16, 0, 16, 1) == -1 and c(16, 16, 0, 1) == -1
    assert c(16, 16, 16, -1) == -1
    assert c(16, 16, 16, 1, precision=7) == -1
    for flags in (dfft.DRY_RUN, dfft.NO_FUSE, dfft.NATURAL_SPECTRUM, dfft.SCALE_BACKWARD | 1, 1 << 31):
        assert c(16, 16, 16, 2, flags=flags) == -1, flags
    for mc in (0, 2, 5, -1):
        assert c(16, 16, 16, 4, mult_count=mc) == -1, mc
    if real:
        assert c(1, 4, 4, 1) == -3
    assert c(4, 4, 512, 1) == 0
    monkeypatch.setenv("DFFT_VARIANT", "5")                  # an alternate tuning of 512: no convolve kernel
    assert c(4, 4, 512, 1) == -3
    monkeypatch.delenv("DFFT_VARIANT")
    monkeypatch.setenv("DFFT_GENERIC", "1")                  # run-time-scheduled entries have no convolve kernel
    assert c(16, 16, 16, 1) == -3
