"""The R2C / C2R convention against the reference tree's heFFTe (heffte::fft3d_r2c, tests/golden/heffte_r2c_vectors.npz).

The committed vectors must equal numpy's rfftn / irfftn * N, and the recorded schedules of dfft_plan_r2c_3d (DRY_RUN plans
interpreted as in test_r2c_dry_run.py) must give the same world arrays for the same P.  Where oracle/_ref/libheffte_r2c_ref.so
is built, the vectors are recomputed with it and must match the committed ones."""
import os
import sys

import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_r2c_dry_run import simulate, x_slabs, y_slabs

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_heffte_r2c_vectors as mk  # noqa: E402


@pytest.fixture(scope="module")
def vectors():
    with np.load(os.path.join(HERE, "golden", "heffte_r2c_vectors.npz")) as z:
        return {k: z[k] for k in z.files}


def test_vectors_cover_the_cases(vectors):
    assert sorted(vectors) == sorted(mk.key(*c) + s for c in mk.CASES for s in ("_fwd", "_bwd"))


@pytest.mark.parametrize("case", mk.CASES, ids=[mk.key(*c) for c in mk.CASES])
def test_heffte_vectors_follow_numpys_convention(vectors, case):
    n0, n1, n2, P = case
    A = mk.case_input(*case)
    F, B = vectors[mk.key(*case) + "_fwd"], vectors[mk.key(*case) + "_bwd"]
    ref = np.fft.rfftn(A)
    assert F.shape == ref.shape and np.abs(F - ref).max() <= 1e-13 * np.abs(ref).max()
    assert B.shape == A.shape and np.abs(B - A * A.size).max() <= 1e-13 * A.size * np.abs(A).max()


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("case", mk.CASES, ids=[mk.key(*c) for c in mk.CASES])
def test_recorded_schedules_equal_heffte(vectors, case, mode):
    n0, n1, n2, P = case
    flags = dfft.EXCHANGE_P2P if mode == "p2p" else dfft.EXCHANGE_NCCL
    A = mk.case_input(*case)
    F, B = vectors[mk.key(*case) + "_fwd"], vectors[mk.key(*case) + "_bwd"]
    got, _, _ = simulate(n0, n1, n2, P, dfft.FORWARD, x_slabs(A, P), flags)
    for d, want in enumerate(y_slabs(F, P)):
        assert np.abs(got[d] - want).max() <= 1e-12 * np.abs(F).max(), (d, "forward")
    got, _, _ = simulate(n0, n1, n2, P, dfft.BACKWARD, y_slabs(np.fft.rfftn(A), P), flags)
    for d, want in enumerate(x_slabs(B, P)):
        assert np.abs(got[d] - want).max() <= 1e-12 * np.abs(B).max(), (d, "backward")


def test_live_heffte_reproduces_the_committed_vectors(vectors):
    from oracle.heffte_r2c import HeffteR2CRef, build_ref_r2c
    if build_ref_r2c() is None:
        pytest.skip("oracle/_ref/libheffte_r2c_ref.so is not built here (the reference tree is absent); the committed vectors are checked above")
    ref = HeffteR2CRef()
    for case in mk.CASES:
        r = mk.compute(ref, *case)
        for s in ("fwd", "bwd"):
            v = vectors[mk.key(*case) + "_" + s]
            assert np.abs(r[s] - v).max() <= 1e-14 * np.abs(v).max(), (case, s)
