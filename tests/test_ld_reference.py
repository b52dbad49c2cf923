"""The long-double FFT of tests/ldfft.py, which the TMA kernel tests use as their reference, and the error metric they apply:
the helper agrees with numpy to fp64 rounding, reproduces closed forms, and the metric's bounds accept a correct fp64 FFT
but reject one whose twiddles in a single stage carry a 40-bit mantissa (an error that the older bound of
1e-12 * log2(N) relative L-infinity against numpy lets through)."""
import numpy as np
import pytest

import ldfft

LENGTHS = [6, 12, 512, 768, 1024]


def _rand(shape, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def test_long_double_is_wider_than_double():
    assert np.finfo(np.longdouble).eps <= ldfft.LD_EPS_MAX


@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("sign", [-1, 1])
def test_agrees_with_numpy_1d(n, sign):
    x = _rand(n, n)
    ref = np.fft.fft(x) if sign < 0 else np.fft.ifft(x) * n
    assert ldfft.errors(ref, ldfft.fft(x, sign=sign))[0] <= 1e-15


@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_agrees_with_numpy_3d(n, axis):
    shape = [4, 6, 8]
    shape[axis] = n
    x = _rand(shape, 10 + n)
    assert ldfft.errors(np.fft.fft(x, axis=axis), ldfft.fft(x, axis=axis))[0] <= 1e-15
    if axis == 0:
        assert ldfft.errors(np.fft.fftn(x), ldfft.fftn(x))[0] <= 1e-15
        assert ldfft.errors(np.fft.ifftn(x) * x.size, ldfft.fftn(x, sign=1))[0] <= 1e-15


@pytest.mark.parametrize("n", LENGTHS)
def test_closed_forms(n):
    eps = 4 * np.finfo(np.longdouble).eps
    d = np.zeros(n, dtype=np.clongdouble)
    d[0] = 1
    assert np.max(np.abs(ldfft.fft(d) - 1)) <= eps                     # impulse -> flat spectrum
    j = np.arange(n)
    for b in (1, n - 1):
        e = ldfft._expi(b * j, n, +1)                                   # e^{2 pi i b j / N} -> N at bin b, 0 elsewhere
        want = np.zeros(n, dtype=np.clongdouble)
        want[b] = n
        assert np.max(np.abs(ldfft.fft(e) - want)) <= n * eps


def _old_bound_passes(got, ref, n):
    # what the fp64 tests accepted before: relative L-infinity against numpy <= 1e-12 * log2(N)
    return np.max(np.abs(got - ref)) / np.max(np.abs(ref)) <= 1e-12 * np.log2(n)


@pytest.mark.parametrize("shape", [(16, 512, 64), (8, 12, 1024), (6, 768, 8)])
def test_metric_accepts_numpy_and_rejects_a_40_bit_twiddle_stage(shape):
    x = _rand(shape, 3)
    ref = ldfft.fftn(x)
    ntot = x.size
    eps = ldfft.EPS["double"]
    r = ldfft.ratios(np.fft.fftn(x), ref, eps, ntot)
    print("numpy fftn", shape, "rel_l2 %.3f linf %.3f (x eps log2 Ntot)" % r)
    assert r[0] <= ldfft.REL_L2_K and r[1] <= ldfft.LINF_K
    exact = ldfft.fftn(x, dtype=np.complex128)                          # the same algorithm in fp64 passes too
    r_exact = ldfft.ratios(exact, ref, eps, ntot)
    assert r_exact[0] <= ldfft.REL_L2_K and r_exact[1] <= ldfft.LINF_K
    bad = ldfft.fftn(x, dtype=np.complex128, perturb=(1, 40))           # one stage of the long axis with 40-bit twiddles
    r_bad = ldfft.ratios(bad, ref, eps, ntot)
    print("40-bit twiddle stage", shape, "rel_l2 %.1f linf %.1f" % r_bad)
    assert r_bad[0] > ldfft.REL_L2_K and r_bad[1] > ldfft.LINF_K
    assert _old_bound_passes(bad, np.fft.fftn(x), ntot)
