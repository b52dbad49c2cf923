"""CPU tests of the batched 3-D lines plans (dfft_lines_plan_create_3d / _r2c_3d) without a GPU.

dfft_debug_lines_3d_ops records the passes a 3-D lines plan launches.  They are interpreted with the slab tests' interpreters
(run_pass for the C2C passes, run_real for the real passes) plus run_plane below for the plane kernel's "XY_PLANE" record, and
the result is compared with numpy's fftn / ifftn * N and rfftn / irfftn * N over axes (1, 2, 3).  Buffers start NaN-filled
with canaries past their ends, so a read or write outside a buffer shows up.  The kernels' arithmetic, and the plane kernel's
bitwise agreement with the separate passes, are checked on the GPU by test_gpu_lines3d.py."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_dry_run import BUF1, IN, MID, OUT, decode, run_pass
from test_r2c_dry_run import run_real
from test_real_lines_dry_run import CANARY, PAD, RealMachine, bufid

TEMP = MID
PLANE_LENGTHS = (16, 32, 64)


def run_plane(m, op):
    """XY_PLANE: for each of ntiles planes, the 2-D transform of the N x N block at in + a*SA (rows cs apart, points es apart)"""
    N = op["N"]
    SAi, _, csi, esi = op["ia"]
    SAo, _, cso, eso = op["oa"]
    y, x = np.meshgrid(np.arange(N), np.arange(N), indexing="ij")
    src, soff = m.view(op["in"])
    dst, doff = m.view(op["out"])
    for a in range(op["ntiles"]):
        blk = src[soff + a * SAi + y * csi + x * esi]
        dst[doff + a * SAo + y * cso + x * eso] = np.fft.ifft2(blk) * N * N if op["inv"] else np.fft.fft2(blk)


def c2c_ops(nx, ny, nz, batch, direction, precision=dfft.DOUBLE):
    return dfft.lines_3d_ops(nx, ny, nz, batch, direction, precision)


def simulate_c2c(nx, ny, nz, batch, direction, data, precision=dfft.DOUBLE):
    count = nx * ny * nz * batch
    m = RealMachine({BUF1: count})
    m.mem[BUF1][:count] = data.reshape(-1)
    m.mem[BUF1].view(np.float64)[2 * count:] = CANARY
    ops = c2c_ops(nx, ny, nz, batch, direction, precision)
    for op in ops:
        assert bufid(op["in"]) == BUF1 and bufid(op["out"]) == BUF1, op["op"]
        run_plane(m, op) if op["op"] == "XY_PLANE" else run_pass(m, op)
    assert np.all(m.mem[BUF1].view(np.float64)[2 * count:] == CANARY), "write past the end of the data"
    got = m.mem[BUF1][:count].copy()
    assert not np.isnan(got.view(np.float64)).any(), "an element was never written (or read NaN)"
    return got, ops


def check(got, want):
    assert got.shape == want.reshape(-1).shape
    assert np.abs(got - want.reshape(-1)).max() <= 1e-11 * max(1.0, np.abs(want).max())


# (nx, ny, nz, batch): the plane lengths; non-square; generic (14, 22, 26), odd (9, 125, 21) and mixed-radix (12, 24, 48, 96)
# lengths; batch 1, odd, and ragged against every tile size
SHAPES = [(16, 16, 16, 3), (32, 32, 8, 2), (64, 64, 4, 1), (16, 16, 5, 7), (32, 32, 3, 5),
          (16, 8, 4, 3), (8, 16, 16, 2), (48, 48, 4, 1), (12, 24, 6, 3), (9, 9, 9, 2), (14, 22, 26, 1), (21, 10, 12, 3),
          (125, 6, 5, 1), (96, 4, 3, 2), (64, 32, 16, 1), (2, 3, 2, 5)]


@pytest.mark.parametrize("nx,ny,nz,batch", SHAPES)
def test_c2c_schedules_match_numpy(nx, ny, nz, batch):
    rng = np.random.default_rng(nx * 10007 + ny * 101 + nz * 7 + batch)
    a = rng.standard_normal((batch, nz, ny, nx)) + 1j * rng.standard_normal((batch, nz, ny, nx))
    plane = nx == ny and nx in PLANE_LENGTHS
    got, ops = simulate_c2c(nx, ny, nz, batch, dfft.FORWARD, a)
    assert [o["op"] for o in ops] == (["XY_PLANE", "Y"] if plane else ["Z", "Y", "Y"])
    check(got, np.fft.fftn(a, axes=(1, 2, 3)))
    got, ops = simulate_c2c(nx, ny, nz, batch, dfft.BACKWARD, a)
    assert [o["op"] for o in ops] == (["Y", "XY_PLANE"] if plane else ["Y", "Y", "Z"])
    check(got, np.fft.ifftn(a, axes=(1, 2, 3)) * nx * ny * nz)


@pytest.mark.parametrize("n", PLANE_LENGTHS)
@pytest.mark.parametrize("precision", [dfft.DOUBLE, dfft.FLOAT])
def test_plane_kernel_is_recorded_exactly_for_its_instantiations(n, precision, monkeypatch):
    for direction in (dfft.FORWARD, dfft.BACKWARD):
        ops = c2c_ops(n, n, 3, 5, direction, precision)
        planes = [o for o in ops if o["op"] == "XY_PLANE"]
        assert len(planes) == 1 and planes[0]["N"] == n and planes[0]["ntiles"] == 15 and planes[0]["inv"] == (direction == dfft.BACKWARD)
    for env in ("DFFT_NO_PLANE", "DFFT_GENERIC"):
        monkeypatch.setenv(env, "1")
        assert [o["op"] for o in c2c_ops(n, n, 3, 5, dfft.FORWARD, precision)] == ["Z", "Y", "Y"], env
        monkeypatch.delenv(env)
    # no plane kernel for other lengths, non-square planes, or real plans
    for shape in ((n, n // 2, 4, 2), (n // 2, n, 4, 2), (128, 128, 2, 1), (48, 48, 2, 1), (n - 4, n - 4, 2, 1)):
        assert all(o["op"] != "XY_PLANE" for o in c2c_ops(*shape, dfft.FORWARD, precision)), shape
    for direction in (dfft.FORWARD, dfft.BACKWARD):
        assert all(o["op"] != "XY_PLANE" for o in dfft.lines_3d_ops(n, n, 4, 2, direction, precision, real=True))


def simulate_real(nx, ny, nz, batch, direction, data, precision=dfft.DOUBLE):
    H = nx // 2 + 1
    rows = ny * nz * batch
    rc, cc = rows * nx, rows * H
    fwd = direction == dfft.FORWARD
    ops = dfft.lines_3d_ops(nx, ny, nz, batch, direction, precision, real=True)
    m = RealMachine({IN: -(-rc // 2) if fwd else cc, OUT: cc if fwd else -(-rc // 2), TEMP: cc})
    (m.mem[IN].view(np.float64) if fwd else m.mem[IN])[: data.size] = data.reshape(-1)
    used_out = 2 * cc if fwd else rc
    m.mem[OUT].view(np.float64)[used_out:] = CANARY
    m.mem[TEMP].view(np.float64)[2 * cc:] = CANARY
    before_in = m.mem[IN].copy()
    for op in ops:
        assert bufid(op["out"]) != IN, ("a pass writes the caller's input", op["op"])
        run_real(m, op) if op["op"] in ("Z_R2C", "Z_C2R") else run_pass(m, op)
    assert np.array_equal(m.mem[IN], before_in, equal_nan=True), "the input buffer was written"
    ov = m.mem[OUT].view(np.float64)
    assert np.all(ov[used_out:] == CANARY), "write past the end of out"
    assert np.all(m.mem[TEMP].view(np.float64)[2 * cc:] == CANARY), "write past the end of the temporary"
    got = m.mem[OUT][:cc].copy() if fwd else ov[:rc].copy()
    assert not np.isnan(got.view(np.float64)).any(), "an output element was never written (or read NaN)"
    return got, ops


# tuned even / odd nx, generic nx, odd and generic ny / nz, batch 1 and odd
REAL_SHAPES = [(16, 16, 16, 3), (64, 8, 4, 1), (9, 8, 6, 3), (14, 12, 10, 2), (21, 10, 3, 1), (22, 26, 5, 3), (125, 6, 4, 2), (2, 3, 5, 1)]


@pytest.mark.parametrize("nx,ny,nz,batch", REAL_SHAPES)
def test_real_schedules_match_numpy(nx, ny, nz, batch):
    rng = np.random.default_rng(nx * 1000 + ny * 10 + nz + batch)
    H = nx // 2 + 1
    a = rng.standard_normal((batch, nz, ny, nx))
    got, ops = simulate_real(nx, ny, nz, batch, dfft.FORWARD, a)
    assert [o["op"] for o in ops] == ["Z_R2C", "Y", "Y"]
    assert all(TEMP not in (bufid(o["in"]), bufid(o["out"])) for o in ops), "the forward schedule uses the temporary"
    check(got, np.fft.rfftn(a, axes=(1, 2, 3)))
    S = rng.standard_normal((batch, nz, ny, H)) + 1j * rng.standard_normal((batch, nz, ny, H))   # not Hermitian
    got, ops = simulate_real(nx, ny, nz, batch, dfft.BACKWARD, S)
    assert [o["op"] for o in ops] == ["Y", "Y", "Z_C2R"]
    assert [(bufid(o["in"]), bufid(o["out"])) for o in ops] == [(IN, TEMP), (TEMP, TEMP), (TEMP, OUT)]
    assert ops[0]["N"] == nz and ops[1]["N"] == ny
    check(got, np.fft.irfftn(S, s=(nz, ny, nx), axes=(1, 2, 3)) * nx * ny * nz)


def code(fn, *args, **kw):
    try:
        fn(*args, **kw)
    except dfft.DfftError as e:
        return int(str(e).split("(")[1].split(")")[0])
    return 0


@pytest.mark.parametrize("real", [False, True])
def test_unsupported_requests_are_refused(real):
    def c(nx, ny, nz, batch, direction=dfft.FORWARD, precision=dfft.DOUBLE):
        return code(dfft.lines_3d_ops, nx, ny, nz, batch, direction, precision, real)
    assert c(16, 16, 16, 4) == 0 and c(14, 22, 26, 1) == 0 and c(16, 16, 16, 0) == 0
    assert c(17, 16, 16, 1) == -3 and c(16, 17, 16, 1) == -3 and c(16, 16, 17, 1) == -3     # prime factor 17
    assert c(8192, 4, 4, 1) == -3                    # nx beyond one shared-memory line (C2C: a four-step 1-D length only)
    assert c(16, 8192, 4, 1) == -3 and c(16, 4, 8192, 1) == -3
    assert c(16, 1, 16, 1) == -3 and c(16, 16, 1, 1) == -3     # no strided pass of length 1
    assert c(16, 16, 16, 1 << 23) == -3 and c(16, 16, 16, (1 << 23) - 1) == 0                # 2^31 rows
    assert c(16, 16, 16, 1 << 62) == -3
    assert c(0, 16, 16, 1) in (-1, -3) and c(16, 0, 16, 1) == -1 and c(16, 16, 0, 1) == -1
    assert c(16, 16, 16, -1) == -1
    assert c(16, 16, 16, 1, direction=0) == -1
    assert c(16, 16, 16, 1, precision=7) == -1
    if real:
        assert c(1, 4, 4, 1) == -3
    else:
        assert c(0, 16, 16, 1) == -1


@pytest.mark.parametrize("precision", [dfft.DOUBLE, dfft.FLOAT])
def test_single_precision_and_forced_generic_schedules(precision, monkeypatch):
    """fp32 entries tile differently; DFFT_GENERIC=1 runs every axis on the run-time-scheduled entries -- same results"""
    rng = np.random.default_rng(5)
    a = rng.standard_normal((3, 6, 32, 32)) + 1j * rng.standard_normal((3, 6, 32, 32))
    got, _ = simulate_c2c(32, 32, 6, 3, dfft.FORWARD, a, precision)
    check(got, np.fft.fftn(a, axes=(1, 2, 3)))
    monkeypatch.setenv("DFFT_GENERIC", "1")
    got, ops = simulate_c2c(32, 32, 6, 3, dfft.BACKWARD, a, precision)
    assert [o["op"] for o in ops] == ["Y", "Y", "Z"]
    check(got, np.fft.ifftn(a, axes=(1, 2, 3)) * 32 * 32 * 6)
    r = rng.standard_normal((2, 5, 12, 64))
    got, _ = simulate_real(64, 12, 5, 2, dfft.FORWARD, r, precision)
    check(got, np.fft.rfftn(r, axes=(1, 2, 3)))
