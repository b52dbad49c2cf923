"""Edge cases of the TMA ring (fft_tma.cuh, tma_ring) under the fused forward t0 (fft_tma_fused_zy_kernel): fewer planes
than the lag, every lag from 1 to 6, and plane counts that leave some CTAs' rings with one ticket more than others.  The
ring's stores stay pending while later tiles land, its slots are freed in order and its end marker must reach every
consumer group.  The kernel runs the same butterflies in the same order as the register-staged sweeps, so every result
must equal the NO_FUSE | NO_TMA plan's bit for bit."""
import faulthandler
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
from gpu_helpers import run_slab  # noqa: E402
from oracle import FORWARD  # noqa: E402

REF_FLAGS = dfft.NO_FUSE | dfft.NO_TMA


@pytest.fixture(autouse=True)
def _watchdog():
    # a host-side hang inside libdfft.so cannot be interrupted by a Python-level signal handler
    faulthandler.dump_traceback_later(240, exit=True, file=sys.stderr)
    yield
    faulthandler.cancel_dump_traceback_later()


def _input(shape, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).reshape(-1)


def _bitwise(shape, seed):
    x = _input(shape, seed)
    got = run_slab(*shape, 1, FORWARD, [x], repeat=2, refill=False)
    ref = run_slab(*shape, 1, FORWARD, [x], flags=REF_FLAGS)
    return got[0], ref[0]


@pytest.mark.parametrize("n0", [2, 4])
def test_fused_t0_fewer_planes_than_the_lag_bitwise(n0, monkeypatch):
    monkeypatch.delenv("DFFT_TMA", raising=False)
    for lag in (n0 + 1, 6):
        monkeypatch.setenv("DFFT_LAG", str(lag))
        got, ref = _bitwise((n0, 512, 512), seed=n0)
        assert got["fused"] == 1 and not ref["fused"]
        assert np.array_equal(got["buf2"], ref["buf2"]), (n0, lag)


@pytest.mark.parametrize("n0", [24, 33])   # 3072 tickets, not a multiple of 132 CTAs; 4224 = 132 * 32
def test_fused_t0_every_lag_bitwise(n0, monkeypatch):
    monkeypatch.delenv("DFFT_TMA", raising=False)
    shape = (n0, 512, 512)
    x = _input(shape, 3)
    ref = run_slab(*shape, 1, FORWARD, [x], flags=REF_FLAGS)[0]
    for lag in range(1, 7):
        monkeypatch.setenv("DFFT_LAG", str(lag))
        got = run_slab(*shape, 1, FORWARD, [x], repeat=2)[0]
        assert got["fused"] == 1
        assert np.array_equal(got["buf2"], ref["buf2"]), lag
