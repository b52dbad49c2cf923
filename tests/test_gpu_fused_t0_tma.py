"""The TMA-pipelined fused forward t0 (fft_tma_fused_zy_kernel: Z and Y roles, intermediate in L2) is the default for
512-point fp64 planes on one device.  It runs the same butterflies in the same order as the register-staged passes, so
every result must equal the NO_FUSE | NO_TMA plan's bit for bit: over several plane counts, repeated executes (the
per-plane counters are monotonic and the ticket counter is re-armed by the last CTA), in place, and with two plans
executed alternately on one device."""
import faulthandler
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
from gpu_helpers import run_slab  # noqa: E402
from oracle import FORWARD  # noqa: E402

N = 512
REF_FLAGS = dfft.NO_FUSE | dfft.NO_TMA


@pytest.fixture(autouse=True)
def _watchdog():
    # a host-side hang inside libdfft.so cannot be interrupted by a Python-level signal handler
    faulthandler.dump_traceback_later(240, exit=True, file=sys.stderr)
    yield
    faulthandler.cancel_dump_traceback_later()


def _input(n0, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((n0, N, N)) + 1j * rng.standard_normal((n0, N, N))).reshape(-1)


@pytest.mark.parametrize("n0", [2, 3, 24, 512])   # 2 and 3 planes: fewer than the default lag
def test_default_t0_is_the_tma_fused_kernel_and_bitwise_the_register_staged_sweeps(n0):
    a = _input(n0, 100 + n0)
    got = run_slab(n0, N, N, 1, FORWARD, [a], repeat=3, refill=False)
    ref = run_slab(n0, N, N, 1, FORWARD, [a], flags=REF_FLAGS)
    assert got[0]["fused"] == 1 and got[0]["launches"] == 2
    assert not ref[0]["fused"] and ref[0]["launches"] == 3
    assert np.array_equal(got[0]["buf2"], ref[0]["buf2"]), n0
    assert np.array_equal(got[0]["buf1"], a[: got[0]["buf1"].size])    # out of place: the input survives


def test_in_place_plan():
    n0 = 8
    a = _input(n0, 7)
    got = run_slab(n0, N, N, 1, FORWARD, [a], repeat=2, inplace=True)
    ref = run_slab(n0, N, N, 1, FORWARD, [a], flags=REF_FLAGS, inplace=True)
    assert got[0]["fused"] == 1
    assert np.array_equal(got[0]["buf2"], ref[0]["buf2"])


def test_two_plans_executed_alternately_on_one_device():
    n0 = 16
    xs = [_input(n0, 11), _input(n0, 12)]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    ins = [torch.from_numpy(x).to(dev) for x in xs]
    outs = [torch.zeros_like(t) for t in ins]
    torch.cuda.synchronize(dev)
    plans = [dfft.fft_mpi_plan_dft_c2c_3d(n0, N, N, ins[k].data_ptr(), outs[k].data_ptr(), None, 0, 1, FORWARD) for k in range(2)]
    assert all(p.fused == 1 for p in plans)
    for _ in range(3):
        for p in plans:
            p.execute()
    for p in plans:
        p.synchronize()
    got = [o.cpu().numpy() for o in outs]
    for p in plans:
        p.destroy()
    for k in range(2):
        ref = run_slab(n0, N, N, 1, FORWARD, [xs[k]], flags=REF_FLAGS)
        assert np.array_equal(got[k], ref[0]["buf2"]), k
