"""CPU tests of the real lines plans (dfft_lines_plan_create_r2c / _r2c_2d) without a GPU.

dfft_debug_real_lines_ops records the passes a real lines plan launches.  They are interpreted here with the interpreters of the
slab tests: run_pass (test_dry_run.py) for the strided C2C pass along ny, run_real (test_r2c_dry_run.py) for the real passes,
and the result is compared with numpy's rfft / irfft * n and rfft2 / irfft2 * nx * ny.  The backward input is not Hermitian.
Every buffer is viewed both as complex128 and as float64; `out` and the temporary start NaN-filled with canaries past their
ends and `in` is NaN past its end, so a read or write outside a buffer, or complex data where real data belongs, shows up.  The
kernels' arithmetic is checked on the GPU by test_gpu_real_lines.py."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_dry_run import IN, MID, OUT, decode, run_pass
from test_r2c_dry_run import run_real

TEMP = MID            # the plan's temporary is symbolic buffer 4
CANARY = 7.25e33
PAD = 64              # complex elements past every buffer's end


class RealMachine:
    """device 0 only: `in`, `out` and the temporary as complex128 arrays of given lengths + PAD"""

    def __init__(self, sizes):
        self.mem = {b: np.full(n + PAD, np.nan, dtype=np.complex128) for b, n in sizes.items()}

    def buf(self, dev, b):
        assert dev == 0, dev
        return self.mem[b]

    def view(self, addr):
        dev, b, off = decode(addr)
        return self.buf(dev, b), off


def bufid(addr):
    return (addr >> 40) & 0xF


def simulate(n, nlines, direction, data, two_d=None, precision=dfft.DOUBLE):
    """data: (nlines, n) reals (forward) or (nlines, n//2+1) complex (backward), nlines = ny*batch rows for 2-D"""
    H = n // 2 + 1
    ops = dfft.real_lines_ops(n, nlines, direction, precision, two_d)
    rows = nlines if two_d is None else two_d[1] * two_d[2]
    rc, cc = rows * n, rows * H
    fwd = direction == dfft.FORWARD
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


def check(got, want):
    assert got.shape == want.reshape(-1).shape
    assert np.abs(got - want.reshape(-1)).max() <= 1e-12 * max(1.0, np.abs(want).max())


# tuned (16, 64, 9, 125, 6, 10) and run-time-scheduled (14, 21, 22, 26, 2, 3, 13) lengths; odd and even
LENGTHS_1D = [(16, 2), (64, 2), (9, 2), (125, 2), (6, 2), (10, 2), (14, 1), (21, 1), (22, 1), (26, 1), (2, 1), (3, 1), (13, 1)]


@pytest.mark.parametrize("n,kind", LENGTHS_1D)
@pytest.mark.parametrize("nlines", [1, 7, 2 * 8 * 3 + 5])
def test_1d_schedules_match_numpy(n, kind, nlines):
    assert dfft.length_kind(n) == kind
    rng = np.random.default_rng(n * 100 + nlines)
    H = n // 2 + 1
    x = rng.standard_normal((nlines, n))
    got, ops = simulate(n, nlines, dfft.FORWARD, x)
    assert [o["op"] for o in ops] == ["Z_R2C"]
    check(got, np.fft.rfft(x, axis=1))
    S = rng.standard_normal((nlines, H)) + 1j * rng.standard_normal((nlines, H))
    got, ops = simulate(n, nlines, dfft.BACKWARD, S)
    assert [o["op"] for o in ops] == ["Z_C2R"]
    check(got, np.fft.irfft(S, n=n, axis=1) * n)
    for direction in (dfft.FORWARD, dfft.BACKWARD):
        assert all(TEMP not in (bufid(o["in"]), bufid(o["out"])) for o in dfft.real_lines_ops(n, nlines, direction))


@pytest.mark.parametrize("precision", [dfft.DOUBLE, dfft.FLOAT])
def test_1d_schedules_single_precision_tiles(precision):
    """fp32 entries tile differently (C); the records are interpreted the same way"""
    for n in (768, 24, 30):
        rng = np.random.default_rng(n)
        x = rng.standard_normal((37, n))
        got, _ = simulate(n, 37, dfft.FORWARD, x, precision=precision)
        check(got, np.fft.rfft(x, axis=1))


# (nx, ny, batch): odd tuned nx, generic nx, generic ny, odd batch
SHAPES_2D = [(9, 8, 3), (16, 12, 1), (14, 12, 2), (16, 14, 3), (21, 10, 1), (22, 26, 3), (125, 6, 2)]


@pytest.mark.parametrize("nx,ny,batch", SHAPES_2D)
def test_2d_schedules_match_numpy(nx, ny, batch):
    rng = np.random.default_rng(nx * 1000 + ny * 10 + batch)
    H = nx // 2 + 1
    a = rng.standard_normal((batch, ny, nx))
    got, ops = simulate(nx, 0, dfft.FORWARD, a, two_d=(nx, ny, batch))
    assert [o["op"] for o in ops] == ["Z_R2C", "Y"]
    assert all(TEMP not in (bufid(o["in"]), bufid(o["out"])) for o in ops), "the forward 2-D schedule uses the temporary"
    check(got, np.fft.rfft2(a, axes=(1, 2)))
    S = rng.standard_normal((batch, ny, H)) + 1j * rng.standard_normal((batch, ny, H))
    got, ops = simulate(nx, 0, dfft.BACKWARD, S, two_d=(nx, ny, batch))
    assert [o["op"] for o in ops] == ["Y", "Z_C2R"]
    assert bufid(ops[0]["in"]) == IN and bufid(ops[0]["out"]) == TEMP and bufid(ops[1]["in"]) == TEMP and bufid(ops[1]["out"]) == OUT
    check(got, np.fft.irfft2(S, s=(ny, nx), axes=(1, 2)) * nx * ny)


def test_unsupported_requests_are_refused():
    def code(*args, two_d=None, precision=dfft.DOUBLE, direction=dfft.FORWARD):
        try:
            dfft.real_lines_ops(*args, direction, precision, two_d)
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0])
        return 0
    assert code(16, 4) == 0 and code(14, 4) == 0
    assert code(17, 4) == -3                                  # prime factor 17
    assert code(1, 4) == -3 and code(0, 4) == -3              # n < 2
    assert code(8192, 4) == -3                                # beyond one shared-memory line in fp64 (a four-step C2C length)
    assert code(6400, 4) == 0 and code(12800, 4, precision=dfft.FLOAT) == 0 and code(12800, 4) == -3
    assert code(16, 1 << 31) == -3 and code(16, (1 << 31) - 1) == 0
    assert code(0, 0, two_d=(16, 1 << 16, 1 << 15)) == -3    # ny * batch rows >= 2^31
    assert code(0, 0, two_d=(16, 17, 2)) == -3                # ny without a strided C2C pass
    assert code(0, 0, two_d=(17, 16, 2)) == -3
    assert code(16, -1) == -1
    assert code(16, 4, direction=0) == -1
    assert code(16, 4, precision=7) == -1


def test_forced_generic_kernel_schedule(monkeypatch):
    """DFFT_GENERIC=1: a tuned length runs on the run-time-scheduled entry (its C), with the same result"""
    plain = dfft.real_lines_ops(64, 9, dfft.FORWARD)
    monkeypatch.setenv("DFFT_GENERIC", "1")
    forced = dfft.real_lines_ops(64, 9, dfft.FORWARD)
    assert plain[0]["C"] != forced[0]["C"]
    x = np.random.default_rng(1).standard_normal((9, 64))
    got, _ = simulate(64, 9, dfft.FORWARD, x)
    check(got, np.fft.rfft(x, axis=1))
