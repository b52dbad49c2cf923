"""CPU tests of the batched 2-D convolve lines plans (dfft_lines_plan_create_convolve_2d / _r2c_2d) without a GPU.

dfft_debug_lines_conv_2d_ops records the passes one execute launches.  They are interpreted with the interpreters of the other
dry-run tests (run_pass for the C2C row passes, run_real for the real row passes, run_xconv for the column pass that transforms
along y, multiplies and transforms back) plus run_plane_conv below for the kernel that convolves whole square images.  The
result is compared with numpy's ifft2(fft2(a) * m) * N and irfft2(rfft2(a) * m) * N, for a multiplier shared by every image
and one per image, scaled and unscaled, in place and out of place.  Every buffer starts NaN-filled with canaries past its end,
so a read outside a buffer, a missed store or a write past an end shows up; `in` (when distinct) and the multiplier must come
back unchanged.  The kernels' arithmetic is checked on the GPU by test_gpu_lines_conv2d.py."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_dry_run import IN, OUT, decode, run_pass  # noqa: F401
from test_lines_conv_dry_run import MULT, TEMP, ConvMachine, check, code, rand_c, run_xconv
from test_r2c_dry_run import run_real
from test_real_lines_dry_run import CANARY, bufid

PLANE_LENGTHS = (16, 32, 64)
PASSES = ["Z", "XCONV", "Z"]


def run_plane_conv(m, op):
    """XY_PLANE_CONV: for each of ntiles images, ifft2(fft2(a) * m) * N^2 (x scale) of the N x N block at in + a*SA (rows cs
    apart, points es apart); the multiplier is N x N in natural order, one for every image when "shared"""
    N = op["N"]
    SAi, _, csi, esi = op["ia"]
    SAo, _, cso, eso = op["oa"]
    y, x = np.meshgrid(np.arange(N), np.arange(N), indexing="ij")
    src, soff = m.view(op["in"])
    dst, doff = m.view(op["out"])
    mul, moff = m.view(op["mult"])
    for a in range(op["ntiles"]):
        blk = src[soff + a * SAi + y * csi + x * esi]
        mk = mul[moff + (0 if op["shared"] else a * N * N) + y * N + x]
        r = np.fft.ifft2(np.fft.fft2(blk) * mk) * N * N
        if op["do_scale"]:
            r = r * op["scale"]
        dst[doff + a * SAo + y * cso + x * eso] = r


def ops_of(nx, ny, batch, real=False, flags=0, mult_count=1, precision=dfft.DOUBLE):
    return dfft.lines_conv_2d_ops(nx, ny, batch, precision, real, flags, mult_count)


def simulate(nx, ny, batch, a, M, real=False, flags=0, inplace=False, precision=dfft.DOUBLE):
    """a: [batch][ny][nx] input; M: the multiplier, one image's (shared) or [batch] of them"""
    H = nx // 2 + 1
    img = nx * ny
    mimg = ny * (H if real else nx)
    mult_count = 1 if M.ndim == 2 else batch
    io = -(-img * batch // 2) if real else img * batch   # complex128 slots holding the caller's buffer
    sizes = {IN: io, OUT: io, MULT: mimg * mult_count}
    if real:
        sizes[TEMP] = ny * H * batch
    m = ConvMachine(sizes, inplace)
    inb = m.mem[IN].view(np.float64) if real else m.mem[IN]
    inb[: a.size] = a.reshape(-1)
    m.mem[MULT][: M.size] = M.reshape(-1)
    keep_in, keep_mult = m.mem[IN].copy(), m.mem[MULT].copy()
    ops = ops_of(nx, ny, batch, real, flags, mult_count, precision)
    for op in ops:
        assert bufid(op["out"]) != MULT and (inplace or bufid(op["out"]) != IN), ("a pass writes a read-only buffer", op["op"])
        if op["op"] == "XY_PLANE_CONV":
            run_plane_conv(m, op)
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
    out = m.mem[OUT].view(np.float64)[: img * batch] if real else m.mem[OUT][: img * batch]
    got = out.copy()
    assert not np.isnan(got.view(np.float64)).any(), "an output element was never written (or read NaN)"
    return got, ops


def want_c2c(a, M, scaled):
    r = np.fft.ifft2(np.fft.fft2(a) * M)
    return r if scaled else r * a.shape[1] * a.shape[2]


def want_r2c(a, M, scaled):
    r = np.fft.irfft2(np.fft.rfft2(a) * M, s=a.shape[1:])
    return r if scaled else r * a.shape[1] * a.shape[2]


# (nx, ny, batch): the plane lengths with whole and partial groups (4 images per CTA at 16, 2 at 32); non-square, generic nx,
# a non-power-of-two square (48, no plane kernel) and odd ny (9, 125)
C2C_SHAPES = [(16, 16, 1), (16, 16, 5), (32, 32, 3), (64, 64, 2), (16, 32, 3), (32, 8, 2), (14, 16, 3), (22, 64, 1),
              (48, 48, 2), (10, 9, 2), (12, 125, 1)]


@pytest.mark.parametrize("nx,ny,batch", C2C_SHAPES)
@pytest.mark.parametrize("env", ["default", "DFFT_NO_PLANE", "DFFT_FORCE_PLANE"])
def test_c2c_convolution_matches_numpy(nx, ny, batch, env, monkeypatch):
    if env != "default":
        monkeypatch.setenv(env, "1")
    rng = np.random.default_rng(nx * 10007 + ny * 101 + batch)
    a = rand_c(rng, (batch, ny, nx))
    M = rand_c(rng, (ny, nx))
    # shared, unscaled, out of place
    got, ops = simulate(nx, ny, batch, a, M)
    seq = [o["op"] for o in ops]
    plane = nx == ny and nx in PLANE_LENGTHS
    if not plane or env == "DFFT_NO_PLANE":
        assert seq == PASSES
    elif env == "DFFT_FORCE_PLANE":
        assert seq == ["XY_PLANE_CONV"]
    else:
        assert seq in (["XY_PLANE_CONV"], PASSES)
    if seq == PASSES:
        assert [o["inv"] for o in ops] == [0, 0, 1]
        assert [(bufid(o["in"]), bufid(o["out"])) for o in ops] == [(IN, OUT), (OUT, OUT), (OUT, OUT)]
        conv = ops[1]
        assert conv["N"] == ny and ops[0]["N"] == nx and ops[2]["N"] == nx
    else:
        conv = ops[0]
        assert (bufid(conv["in"]), bufid(conv["out"])) == (IN, OUT)
        assert conv["N"] == nx and conv["ntiles"] == batch and conv["ia"] == conv["oa"] == [nx * ny, 0, nx, 1]
    assert conv["shared"] == 1 and bufid(conv["mult"]) == MULT and not conv["do_scale"]
    check(got, want_c2c(a, M, False))
    # one per image, scaled, in place
    Mb = rand_c(rng, (batch, ny, nx))
    got, ops = simulate(nx, ny, batch, a, Mb, flags=dfft.SCALE_BACKWARD, inplace=True)
    conv = ops[1] if len(ops) == 3 else ops[0]
    assert conv["shared"] == (batch == 1) and conv["do_scale"] and conv["scale"] == pytest.approx(1.0 / (nx * ny), rel=1e-15)
    check(got, want_c2c(a, Mb, True))
    # one per image, unscaled, out of place
    got, _ = simulate(nx, ny, batch, a, Mb)
    check(got, want_c2c(a, Mb, False))


# tuned even / odd nx, generic nx (14, 21, 15), odd ny, the shortest real line
R2C_SHAPES = [(16, 16, 3), (64, 64, 1), (9, 8, 3), (14, 16, 2), (21, 10, 1), (32, 12, 2), (2, 4, 2), (15, 32, 3), (64, 125, 1)]


@pytest.mark.parametrize("nx,ny,batch", R2C_SHAPES)
def test_r2c_convolution_matches_numpy(nx, ny, batch):
    rng = np.random.default_rng(nx * 1000 + ny * 10 + batch)
    H = nx // 2 + 1
    a = rng.standard_normal((batch, ny, nx))
    M = rand_c(rng, (ny, H))   # not Hermitian: the C2R ignores what numpy's irfft2 ignores
    got, ops = simulate(nx, ny, batch, a, M, real=True)
    assert [o["op"] for o in ops] == ["Z_R2C", "XCONV", "Z_C2R"]
    assert [(bufid(o["in"]), bufid(o["out"])) for o in ops] == [(IN, TEMP), (TEMP, TEMP), (TEMP, OUT)]
    assert ops[1]["N"] == ny and ops[1]["W"] == H and ops[1]["shared"] == 1
    check(got, want_r2c(a, M, False))
    Mb = rand_c(rng, (batch, ny, H))
    for inplace in (False, True):
        got, ops = simulate(nx, ny, batch, a, Mb, real=True, flags=dfft.SCALE_BACKWARD, inplace=inplace)
        assert ops[1]["shared"] == (batch == 1) and ops[1]["do_scale"]   # mult_count == batch == 1 is the shared case
        check(got, want_r2c(a, Mb, True))


@pytest.mark.parametrize("n", PLANE_LENGTHS)
@pytest.mark.parametrize("precision", [dfft.DOUBLE, dfft.FLOAT])
def test_plane_conv_selection(n, precision, monkeypatch):
    """the one-kernel convolution runs where the table says, everywhere under DFFT_FORCE_PLANE=1 and nowhere under
    DFFT_NO_PLANE=1, read from the environment at creation; never for the real plan"""
    def seq(**kw):
        return [o["op"] for o in ops_of(n, n, 5, precision=precision, **kw)]
    assert seq() in (["XY_PLANE_CONV"], PASSES)
    monkeypatch.setenv("DFFT_NO_PLANE", "1")
    assert seq() == PASSES
    monkeypatch.delenv("DFFT_NO_PLANE")
    monkeypatch.setenv("DFFT_FORCE_PLANE", "1")
    assert seq() == ["XY_PLANE_CONV"]
    assert seq(real=True) == ["Z_R2C", "XCONV", "Z_C2R"]
    assert [o["op"] for o in ops_of(n, 2 * n, 5, precision=precision)] == PASSES   # not square


@pytest.mark.parametrize("precision", [dfft.DOUBLE, dfft.FLOAT])
def test_single_precision_schedule_matches_numpy(precision, monkeypatch):
    """fp32 entries tile differently (other C per pass); the schedule is the same arithmetic"""
    rng = np.random.default_rng(11)
    for nx, ny, batch in ((20, 24, 3), (32, 32, 3)):
        a = rand_c(rng, (batch, ny, nx))
        M = rand_c(rng, (ny, nx))
        for env in ("DFFT_NO_PLANE", "DFFT_FORCE_PLANE"):
            monkeypatch.setenv(env, "1")
            got, _ = simulate(nx, ny, batch, a, M, precision=precision)
            monkeypatch.delenv(env)
            check(got, want_c2c(a, M, False))


@pytest.mark.parametrize("real", [False, True])
def test_unsupported_requests_are_refused(real, monkeypatch):
    def c(nx, ny, batch, flags=0, mult_count=1, precision=dfft.DOUBLE):
        return code(ops_of, nx, ny, batch, real, flags, mult_count, precision)
    assert c(16, 16, 4) == 0 and c(14, 16, 1) == 0 and c(16, 16, 0) == 0 and c(16, 16, 4, mult_count=4) == 0
    assert c(16, 16, 4, flags=dfft.SCALE_BACKWARD) == 0
    for ny in (14, 22, 26, 17):                              # no tuned kernel (generic lengths) or no kernel at all
        assert dfft.length_kind(ny, dfft.DOUBLE) != 2
        assert c(16, ny, 1) == -3, ny
    assert c(17, 16, 1) == -3                                # nx without any kernel
    assert c(16, 1, 1) == -3                                 # no strided pass of length 1
    assert c(16, 16, 1 << 27) == -3 and c(16, 16, (1 << 27) - 1) == 0   # 2^31 rows
    assert c(0, 16, 1) in (-1, -3) and c(16, 0, 1) == -1
    assert c(16, 16, -1) == -1
    assert c(16, 16, 1, precision=7) == -1
    for flags in (dfft.DRY_RUN, dfft.NO_FUSE, dfft.NATURAL_SPECTRUM, dfft.SCALE_BACKWARD | 1, 1 << 31):
        assert c(16, 16, 2, flags=flags) == -1, flags
    for mc in (0, 2, 5, -1):
        assert c(16, 16, 4, mult_count=mc) == -1, mc
    if real:
        assert c(1, 4, 1) == -3
    else:
        assert c(1, 16, 1) == -3                             # no C2C line of length 1
    assert c(4, 512, 1) == 0
    monkeypatch.setenv("DFFT_VARIANT", "5")                  # an alternate tuning of 512: no convolve kernel
    assert c(4, 512, 1) == -3
    monkeypatch.delenv("DFFT_VARIANT")
    monkeypatch.setenv("DFFT_GENERIC", "1")                  # run-time-scheduled entries have no convolve kernel
    assert c(16, 16, 1) == -3
