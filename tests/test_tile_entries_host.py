"""CPU test of the register-staged kernel table pinned in tests/tile_entries.py, on the real library without a GPU: a DFFT_DRY_RUN
plan makes no CUDA call and records the passes it would launch (as in test_dry_run.py).  For every default entry and axis, a
NO_TMA | NO_FUSE thin-slab plan must record, for each of its three passes, the pass kind, the length of that axis and the C of that
length's entry: forward Z, Y, XF and backward XB, Y, Z; with NATURAL_SPECTRUM the X pass is a Y pass with the X length's s_C.  A
change to the kernel tables therefore shows up here instead of silently moving test_gpu_tile_matrix.py onto other kernels."""
import pytest

import distributedfft_b200 as dfft
from tile_entries import AXES, BY, DOUBLE, ENTRIES, FLOAT, NOT_FUSED, entry_id, lengths, thin_shape

FLAGS = dfft.NO_TMA | dfft.NO_FUSE


def fake(dev, buf):
    return ((dev + 1) << 44) | (buf << 40)


def recorded(shape, prec, direction, flags):
    p = dfft.fft_mpi_plan_dft_c2c_3d(*shape, fake(0, 5), fake(0, 2), None, 0, 1, direction, prec, flags | dfft.DRY_RUN)
    try:
        p.execute()
        ops, fused = p.recorded_ops(), p.fused
    finally:
        p.destroy()
    assert not fused
    return [(o["op"], o["N"], o["C"]) for o in ops]


def expected(shape, prec, direction, natural):
    """(op, N, C) of the three passes, in launch order"""
    n0, n1, n2 = shape
    z = ("Z", n2, BY[n2, prec][2][0])
    y = ("Y", n1, BY[n1, prec][2][1])
    x = ("Y", n0, BY[n0, prec][2][1]) if natural else ("XF" if direction == dfft.FORWARD else "XB", n0, BY[n0, prec][2][2])
    return [z, y, x] if direction == dfft.FORWARD else [x, y, z]


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["f64", "f32"])
def test_pinned_lengths_are_the_supported_lengths(prec):
    assert lengths(prec) == dfft.supported_lengths(prec)
    for n in lengths(prec):
        assert dfft.length_kind(n, prec) == 2, n
        e = BY[n, prec]
        assert all(n % r == 0 for r in e[3]), e


@pytest.mark.parametrize("entry", ENTRIES, ids=[entry_id(e) for e in ENTRIES])
def test_fused_t0_exists_where_its_roles_fit_in_shared_memory(entry):
    """square planes take the fused register-staged t0 (forced on one device, the P2P default with P > 1) exactly where the entry
    has that kind; where its roles would need more than 227 KB of shared memory the plan keeps the separate passes instead of
    failing at execute"""
    n, prec = entry[0], entry[1]
    missing = NOT_FUSED.get((n, prec), set())
    for P, flags, kinds in ((1, dfft.FORCE_FUSE, ("ZY", "YZ")), (2, dfft.EXCHANGE_P2P, ("ZY_CO", "YZ_CI"))):
        for direction, kind in zip((dfft.FORWARD, dfft.BACKWARD), kinds):
            p = dfft.fft_mpi_plan_dft_c2c_3d(2 * P, n, n, fake(0, 5), fake(0, 2), None, 0, P, direction, prec, flags | dfft.NO_TMA | dfft.DRY_RUN)
            try:
                p.execute()
                names = [o["op"] for o in p.recorded_ops()]
                assert p.fused == (kind not in missing), (kind, names)
                assert ("fusedZ" in names and "fusedY" in names) == p.fused and ("Z" in names) != p.fused, names
            finally:
                p.destroy()


def test_generic_kernel_shared_memory_limits():
    """two copies of a line must fit in 200 KB of shared memory: 6400 points fp64, 12800 fp32 (test_gpu_tile_matrix.py runs both
    limits); the next smooth lengths have no kernel"""
    assert dfft.length_kind(6400, DOUBLE) == 1 and dfft.length_kind(6656, DOUBLE) == 0 and dfft.length_kind(12800, DOUBLE) == 0
    assert dfft.length_kind(12800, FLOAT) == 1 and dfft.length_kind(13000, FLOAT) == 0 and dfft.length_kind(6656, FLOAT) == 1


@pytest.mark.parametrize("entry", ENTRIES, ids=[entry_id(e) for e in ENTRIES])
def test_every_axis_records_the_pinned_pass_and_c(entry):
    n, prec = entry[0], entry[1]
    for axis in (2, 1, 0):
        shape = thin_shape(n, axis)
        for direction in (dfft.FORWARD, dfft.BACKWARD):
            want = expected(shape, prec, direction, False)
            assert recorded(shape, prec, direction, FLAGS) == want, (AXES[axis], direction)
            if axis == 0:
                want = expected(shape, prec, direction, True)
                assert recorded(shape, prec, direction, FLAGS | dfft.NATURAL_SPECTRUM) == want, ("natural X", direction)
