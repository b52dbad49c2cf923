"""CPU tests of the general 1-D layouts of dfft_lines_plan_create: line l at (l / inner) * outer_dist + (l % inner) * inner_dist,
points `stride` apart.  The recorded pass (dfft_debug_lines_ops) is interpreted on a flat buffer whose every element outside the
lines is NaN (test_dry_run.run_pass), for padded rows, gaps between matrices, interleaved matrices, ragged column tiles and the
grouped contiguous form, in both precisions.  The result must match numpy on the lines and leave every other element NaN.
Layouts whose columns would overlap, and negative matrix distances, are DFFT_EINVAL."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_dry_run import BUF1, FlatMachine, fake, run_pass

DOUBLE, FLOAT, FORWARD, BACKWARD = dfft.DOUBLE, dfft.FLOAT, dfft.FORWARD, dfft.BACKWARD
EINVAL, EUNSUPPORTED = r"\(-1\)", r"\(-3\)"


def line_offsets(n, stride, nlines, inner, inner_dist, outer_dist):
    """[nlines][n] element offsets of the points of every line"""
    l = np.arange(nlines)[:, None]
    return (l // inner) * outer_dist + (l % inner) * inner_dist + np.arange(n)[None, :] * stride


# (name, n, stride, nlines, inner, inner_dist, outer_dist)
LAYOUTS = [
    ("padded-rows", 96, 24, 63, 21, 1, 96 * 24),                 # 3 matrices of 96 rows, 21 of 24 columns used
    ("gapped", 64, 10, 30, 10, 1, 64 * 10 + 37),                 # dense rows, 37 elements between matrices
    ("padded-gapped", 48, 40, 66, 33, 1, 48 * 40 + 5),           # both, and 33 columns: ragged for every column tile width
    ("interleaved", 48, 14, 14, 7, 1, 7),                        # two matrices whose rows alternate
    ("interleaved-padded", 100, 17, 15, 5, 1, 5),                # three matrices' rows alternate, then 2 unused per row
    ("ragged-one-matrix", 9, 45, 45, 45, 1, 0),                  # 45 columns of one matrix, outer_dist ignored
    ("one-matrix-negative", 12, 11, 11, 11, 1, -7),              # the same with a negative outer_dist
    ("single-column-gapped", 64, 3, 4, 1, 1, 64 * 3 + 1),        # one column per matrix: stride over unused columns
    ("grouped-contiguous", 64, 1, 24, 8, 64, 8 * 64),            # contiguous lines in groups of 8, densely packed
    ("generic-padded", 14, 9, 21, 7, 1, 14 * 9),                 # a run-time-scheduled length
]


@pytest.mark.parametrize("precision", [DOUBLE, FLOAT], ids=["f64", "f32"])
@pytest.mark.parametrize("name,n,stride,nlines,inner,inner_dist,outer_dist", LAYOUTS, ids=[c[0] for c in LAYOUTS])
def test_layout_transforms_the_lines_and_nothing_else(name, n, stride, nlines, inner, inner_dist, outer_dist, precision):
    off = line_offsets(n, stride, nlines, inner, inner_dist, outer_dist)
    assert off.min() >= 0 and np.unique(off).size == off.size, "the layout itself overlaps"
    size = int(off.max()) + 1 + 19
    rng = np.random.default_rng(n * 1000 + nlines)
    x = rng.standard_normal((nlines, n)) + 1j * rng.standard_normal((nlines, n))
    untouched = np.ones(size, dtype=bool)
    untouched[off.ravel()] = False
    for direction in (FORWARD, BACKWARD):
        ops = dfft.lines_ops(n, stride, nlines, inner, inner_dist, outer_dist, direction, precision)
        assert len(ops) == 1 and ops[0]["op"] == ("Z" if stride == 1 else "Y"), ops
        if name.startswith(("ragged", "padded-gapped")):
            assert ops[0]["W"] % ops[0]["C"] != 0, ops[0]
        m = FlatMachine(size)
        buf = m.view(fake(0, BUF1))[0]
        buf[:] = complex(np.nan, np.nan)
        buf[off] = x
        run_pass(m, ops[0])
        ref = np.fft.fft(x, axis=1) if direction == FORWARD else np.fft.ifft(x, axis=1) * n
        assert np.abs(buf[off] - ref).max() <= 1e-12 * np.log2(max(n, 2)) * np.abs(ref).max(), (name, direction)
        assert np.isnan(buf[untouched]).all(), "an element outside the lines was written"


def test_dense_layouts_keep_their_records():
    """padding changes only the strides of a pass: tile size, tile and column counts are those of the dense layout"""
    dense = dfft.lines_ops(96, 21, 63, 21, 1, 96 * 21, FORWARD)[0]
    padded = dfft.lines_ops(96, 24, 63, 21, 1, 96 * 24 + 5, FORWARD)[0]
    assert padded["ia"] == padded["oa"] == [96 * 24 + 5, dense["C"], 1, 24], padded
    for k in ("op", "N", "C", "G", "W", "ntiles"):
        assert padded[k] == dense[k], k


# (why, n, stride, nlines, inner, outer_dist): every pair is a layout whose columns touch an element twice
OVERLAPPING = [
    ("more columns than the row holds", 16, 4, 10, 5, 80),
    ("two matrices at one address", 16, 4, 8, 4, 0),
    ("negative matrix distance", 16, 4, 8, 4, -64),
    ("matrices one element too close", 16, 4, 8, 4, 63),
    ("interleaved rows that collide", 16, 8, 8, 4, 3),
    ("interleaved matrix offset past the gap", 16, 8, 8, 4, 6),
    ("three interleaved in room for two", 16, 8, 12, 4, 4),
    ("matrix distance equal to the row stride", 16, 64, 8, 4, 64),
]


@pytest.mark.parametrize("precision", [DOUBLE, FLOAT], ids=["f64", "f32"])
@pytest.mark.parametrize("why,n,stride,nlines,inner,outer_dist", OVERLAPPING, ids=[c[0].replace(" ", "-") for c in OVERLAPPING])
def test_overlapping_column_layouts_are_rejected(why, n, stride, nlines, inner, outer_dist, precision):
    with pytest.raises(dfft.DfftError, match=EINVAL):
        dfft.lines_ops(n, stride, nlines, inner, 1, outer_dist, FORWARD, precision)


def test_the_non_overlap_rule_at_its_edges():
    # the smallest legal matrix distance, interleaved matrices filling every row exactly, a single column per matrix
    for args in ((16, 4, 8, 4, 1, 64), (16, 8, 8, 4, 1, 4), (16, 12, 12, 4, 1, 4), (16, 8, 8, 1, 1, 1), (16, 8, 8, 1, 1, 129)):
        assert [o["op"] for o in dfft.lines_ops(*args, FORWARD)] == ["Y"], args
    # a single column per matrix with the matrices inside one column's span: they overlap
    with pytest.raises(dfft.DfftError, match=EINVAL):
        dfft.lines_ops(16, 8, 8, 1, 1, 8, FORWARD)


def test_long_lines_must_be_densely_packed():
    """the four-step plan addresses its lines as one dense block: the grouped dense form is the plain one, a gap is refused"""
    n = 8192
    dense = dfft.lines_ops(n, 1, 4, 4, n, 0, FORWARD)
    assert [o["op"] for o in dense] == ["XF_TW", "Y"]
    assert dfft.lines_ops(n, 1, 4, 2, n, 2 * n, FORWARD) == dense
    with pytest.raises(dfft.DfftError, match=EUNSUPPORTED):
        dfft.lines_ops(n, 1, 4, 2, n, 3 * n, FORWARD)
