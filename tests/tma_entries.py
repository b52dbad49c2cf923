"""The table of TMA-pipelined kernels (dfft_kernels_tma.cu) as the tests expect it: per (length, precision) the lines per
tile C and the passes that use the TMA kernel by default.  DFFT_TMA=2 turns on every pass mode and keeps the fused forward
t0 (ZY) where the default has it.  test_tma_host_fakecuda.py checks these values against the library without a GPU;
test_gpu_tma_matrix.py runs every (entry, mode) on the GPU."""
DOUBLE, FLOAT = 0, 1
MODES = ("Z", "Y", "XF", "XB")
MASK_BIT = {"Z": 1, "Y": 2, "XF": 4, "XB": 4}   # plan.tma_mask: the X bit follows the plan's direction

# (N, precision, C, modes used by default)
ENTRIES = [
    (512, DOUBLE, 8, {"Y", "XF", "ZY"}),
    (1024, DOUBLE, 4, {"Y", "XF", "XB"}),
    (256, DOUBLE, 16, {"Z", "Y", "XF", "XB"}),
    (768, DOUBLE, 4, {"Y"}),
    (512, FLOAT, 16, {"Z", "Y", "XF", "XB"}),
    (1024, FLOAT, 8, {"Y", "XF", "XB"}),
    (768, FLOAT, 8, {"Y", "XF", "XB"}),
]
TMA_LENGTHS = {e[0] for e in ENTRIES}


def modes(entry, forced):
    """the modes an entry uses by default or under DFFT_TMA=2"""
    used = entry[3]
    return set(MODES) | (used & {"ZY"}) if forced else set(used)


def rows(n):
    return min(n, 256)


def entry_id(entry):
    return "%d%s" % (entry[0], "f64" if entry[1] == DOUBLE else "f32")


def esz(precision):
    return 16 if precision == DOUBLE else 8


def thin_shape(entry, axis, short=(12, 32)):
    """a slab whose only long axis is `axis` (0 = X, 1 = Y, 2 = Z); the short axes are not TMA lengths and keep every
    TMA pass of that axis applicable (n2 a multiple of C, n0*n1 a multiple of C)"""
    n = entry[0]
    a, b = short
    return {2: (a, b, n), 1: (a, n, b), 0: (n, a, b)}[axis]
