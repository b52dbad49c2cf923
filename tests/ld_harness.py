"""The harness of the long-double kernel matrices (test_gpu_tma_matrix.py, test_gpu_tile_matrix.py): seeded or structured inputs
and their long-double references (tests/ldfft.py), cached per (shape, seed, precision, sign, kind, axis); the device layouts of a
P = 1 plan; one plan on fenced, NaN-prefilled buffers executed several times; an in-place lines plan in a fenced layout whose
gaps must stay unchanged; and the two error ratios against the bounds
ldfft.REL_L2_K / ldfft.LINF_K (in units of eps * log2(Ntot))."""
import collections

import numpy as np
import torch

import distributedfft_b200 as dfft
import ldfft

DOUBLE, FLOAT = dfft.DOUBLE, dfft.FLOAT
FWD, BWD = dfft.FORWARD, dfft.BACKWARD
CDT = {DOUBLE: (np.complex128, torch.complex128), FLOAT: (np.complex64, torch.complex64)}
EPS = {DOUBLE: ldfft.EPS["double"], FLOAT: ldfft.EPS["float"]}
CANARY = 48

# ---- inputs and long-double references ------------------------------------------------------------------------------------
_refs = collections.OrderedDict()


def logical_input(shape, seed, prec, sign, kind, axis=None):
    """kind "rand": seeded complex normal; "delta": 1 at the last element of the device buffer in either layout (and of the
    last tile); "expo": one exponential at bin N-1 of `axis` (default: the longest axis), constant along the others"""
    npdt = CDT[prec][0]
    if kind == "rand":
        rng = np.random.default_rng(seed)
        return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(npdt)
    x = np.zeros(shape, dtype=npdt)
    if kind == "delta":
        x[-1, -1, -1] = 1
        return x
    axis = int(np.argmax(shape)) if axis is None else axis
    n = shape[axis]
    e = ldfft._expi((n - 1) * np.arange(n), n, -sign).astype(npdt)
    sl = [None, None, None]
    sl[axis] = slice(None)
    return np.broadcast_to(e[tuple(sl)], shape).astype(npdt)


def reference(shape, seed, prec, sign, kind="rand", axis=None):
    """(input, its long-double 3-D transform of sign `sign`); the last six are kept"""
    key = (tuple(shape), seed, prec, sign, kind, axis)
    if key not in _refs:
        x = logical_input(shape, seed, prec, sign, kind, axis)
        _refs[key] = (x, ldfft.fftn(x, sign=sign))
        while len(_refs) > 6:
            _refs.popitem(last=False)
    _refs.move_to_end(key)
    return _refs[key]


def layouts(shape, seed, prec, direction, kind="rand", natural=False, scale=False, axis=None):
    """(device input, expected output), both flat, for a P = 1 plan: forward [x][y][z] -> [y][z][x], backward the reverse
    (natural spectrum: [x][y][z] both ways)"""
    x, y = reference(shape, seed, prec, -1 if direction == FWD else 1, kind, axis)
    if natural:
        dev_in, want = x.reshape(-1), y.reshape(-1)
    elif direction == FWD:
        dev_in, want = x.reshape(-1), y.transpose(1, 2, 0).reshape(-1)
    else:
        dev_in, want = x.transpose(1, 2, 0).reshape(-1), y.reshape(-1)
    if scale:
        want = want / np.longdouble(x.size)
    return np.ascontiguousarray(dev_in), want


# ---- one plan on its own fenced buffers ----------------------------------------------------------------------------------
def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def run_fenced(shape, prec, direction, dev_in, flags=0, inplace=False, offset=0, repeat=3, info=None):
    """create a P = 1 plan on fresh buffers and execute it `repeat` times; returns (output, tma_mask, fused).  The output
    view starts `offset` elements after a canary block and is followed by another (the arena itself is 256-byte aligned).
    `info`: a dict that also receives the plan's launches per execute."""
    npdt, tdt = CDT[prec]
    n = int(np.prod(shape))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    total = CANARY + offset + n + CANARY
    lo, hi = CANARY + offset, CANARY + offset + n
    rng = np.random.default_rng(12345)
    pattern = np.zeros(total, dtype=npdt)          # random canaries; the output region is refilled below
    pattern[:lo] = rng.standard_normal(lo) + 1j * rng.standard_normal(lo)
    pattern[hi:] = rng.standard_normal(CANARY) + 1j * rng.standard_normal(CANARY)
    arena = torch.from_numpy(pattern).to(dev)
    view = arena[CANARY + offset: CANARY + offset + n]
    if inplace:
        view.copy_(torch.from_numpy(dev_in).to(dev))
        tin = None
    else:
        view.fill_(complex(float("nan"), float("nan")))
        tin = torch.from_numpy(dev_in).to(dev)
    torch.cuda.synchronize(dev)
    plan = dfft.fft_mpi_plan_dft_c2c_3d(*shape, (view if inplace else tin).data_ptr(), None if inplace else view.data_ptr(), None, 0, 1,
                                        direction, prec, flags)
    try:
        outs = []
        for _ in range(repeat):
            plan.execute()
            plan.synchronize()
            outs.append(view.cpu().numpy().copy())
        mask, fused = plan.tma_mask, plan.fused
        if info is not None:
            info["launches"] = plan.launches
    finally:
        plan.destroy()
    got = outs[0]
    assert not np.isnan(got.view(npdt().real.dtype)).any(), "NaN left in the output region: an element was never written"
    assert np.array_equal(bits(arena[:lo].cpu().numpy()), bits(pattern[:lo])), "canary before the output overwritten"
    assert np.array_equal(bits(arena[hi:].cpu().numpy()), bits(pattern[hi:])), "canary after the output overwritten"
    for k in range(1, repeat):
        assert np.array_equal(bits(outs[k]), bits(got)), "execute %d differs from the first" % k
    if tin is not None:
        assert np.array_equal(bits(tin.cpu().numpy()), bits(dev_in)), "out-of-place input modified"
    return got, mask, fused


def run_lines(plan, x, prec, direction, repeat=2, offsets=None, size=None, offset=0):
    """in-place lines plan on a fenced device copy of `x`, executed `repeat` times from the same input; returns the result in x's
    shape.  `offsets` (x's shape, the element offsets of x's points in a buffer of `size` elements, as a layout places them)
    scatter x into that buffer; by default x is dense.  Every element of the arena outside x -- the canaries at both ends and the
    gaps inside the layout -- holds a random pattern that must come back bit for bit.  `offset`: elements between the leading
    canary and the buffer (the arena itself is 256-byte aligned)."""
    npdt = CDT[prec][0]
    if offsets is None:
        offsets, size = np.arange(x.size).reshape(x.shape), x.size
    lo = CANARY + offset
    total = lo + size + CANARY
    pattern = (np.random.default_rng(5).standard_normal(total) * (1 + 1j)).astype(npdt)
    filled = pattern.copy()
    filled[lo + offsets] = x
    dev = torch.device("cuda", 0)
    arena = torch.empty(total, dtype=CDT[prec][1], device=dev)
    outs = []
    for _ in range(repeat):
        arena.copy_(torch.from_numpy(filled))
        torch.cuda.synchronize(dev)                  # the plan runs on its own stream
        plan.execute(arena[lo:].data_ptr(), direction)
        plan.synchronize()
        outs.append(arena.cpu().numpy())
    keep = np.ones(total, dtype=bool)
    keep[lo + offsets] = False
    assert np.array_equal(bits(outs[0][keep]), bits(pattern[keep])), "an element outside the lines (a canary or a gap) was written"
    for o in outs[1:]:
        assert np.array_equal(bits(o), bits(outs[0])), "executes differ"
    return outs[0][lo + offsets]


# ---- the bounds ----------------------------------------------------------------------------------------------------------
def check(tag, got, want, prec, ntot, label, linf_scale="rms"):
    """assert both ratios against the long-double (or clongdouble-castable) reference and print them on a `tag` line"""
    r = ldfft.ratios(got, want, EPS[prec], ntot, linf_scale)
    print("%s %-52s rel_l2 %6.3f  linf %6.3f" % (tag, label, r[0], r[1]))
    assert r[0] <= ldfft.REL_L2_K and r[1] <= ldfft.LINF_K, (label, r)
    return r


def ratios64(got, ref, eps, ntot):
    """ldfft.ratios evaluated in fp64 (full cubes: the long-double copies would need tens of GB); the difference of two fp64
    values this close is exact, so only the reference's own error (scipy, about 0.14 / 0.6 in these units) is added"""
    ref = np.asarray(ref).ravel()
    d = np.abs(np.asarray(got).ravel().astype(ref.dtype) - ref)
    n2 = np.sum(np.abs(ref) ** 2)
    u = eps * np.log2(ntot)
    return float(np.sqrt(np.sum(d ** 2) / n2)) / u, float(d.max() / np.sqrt(n2 / ref.size)) / u
