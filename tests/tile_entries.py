"""The register-staged kernel table (dfft_kernels_f64.cu, dfft_kernels_f32.cu; fft_tile_kernel) as the tests expect it: per default
entry (N, precision) the lines per tile C of the Z (contiguous), Y (strided, local) and X (t3) configurations, and the points per
thread R of their schedules (Sched<N, R, radices...>), so that a CTA has T * C = N / R * C threads.  The library does not report R;
it is taken from the tables.  test_tile_entries_host.py checks the lengths and every C against DRY_RUN plans without a GPU;
test_gpu_tile_matrix.py runs every (entry, pass) on the GPU."""
DOUBLE, FLOAT = 0, 1

# N: (z_C, s_C, x_C), (z_R, s_R, x_R)
_COMMON = {
    4: ((64, 32, 32), (2, 2, 2)),
    8: ((64, 32, 32), (4, 4, 4)),
    16: ((32, 32, 32), (4, 4, 4)),
    32: ((32, 32, 32), (8, 8, 8)),
    64: ((16, 16, 16), (8, 8, 8)),
    128: ((16, 16, 16), (16, 16, 16)),
    256: ((8, 8, 8), (16, 16, 16)),
    512: ((2, 8, 8), (8, 16, 16)),
    2048: ((1, 4, 4), (16, 16, 16)),
    4096: ((1, 2, 2), (16, 16, 16)),
    384: ((4, 8, 8), (12, 12, 12)),
    192: ((8, 8, 8), (12, 12, 12)),
    96: ((16, 16, 16), (12, 12, 12)),
    48: ((32, 32, 32), (12, 12, 12)),
    24: ((32, 32, 32), (6, 6, 6)),
    12: ((64, 32, 32), (6, 6, 6)),
    6: ((64, 32, 32), (6, 6, 6)),
    9: ((32, 32, 32), (3, 3, 3)),
    10: ((64, 32, 32), (10, 10, 10)),
    100: ((16, 16, 16), (10, 10, 10)),
    125: ((8, 8, 8), (5, 5, 5)),
    49: ((16, 16, 16), (7, 7, 7)),
    243: ((8, 8, 8), (9, 9, 9)),
    1000: ((2, 4, 4), (10, 10, 10)),
}
_OWN = {
    DOUBLE: {1024: ((1, 4, 8), (8, 16, 16)), 768: ((4, 4, 4), (24, 24, 24))},
    FLOAT: {1024: ((2, 16, 16), (16, 32, 32)), 768: ((2, 16, 16), (12, 24, 24))},
}

# (N, precision, (z_C, s_C, x_C), (z_R, s_R, x_R))
ENTRIES = [(n, p, c, r) for p in (DOUBLE, FLOAT) for n, (c, r) in sorted({**_COMMON, **_OWN[p]}.items())]
BY = {(e[0], e[1]): e for e in ENTRIES}
# fused register-staged kinds (fft_fused2_kernel) that an entry does not have because their two roles need more than the 227 KB
# of shared memory a block can get: ZY / YZ = one-device forward / backward t0, ZY_CO / YZ_CI = the P > 1 forms with chunk tables
NOT_FUSED = {(4096, DOUBLE): {"ZY", "YZ", "ZY_CO", "YZ_CI"}, (2048, DOUBLE): {"ZY_CO", "YZ_CI"}}
AXES = {2: "Z", 1: "Y", 0: "X"}            # axis of the 3-D array -> pass; X's C and R are the x_ values
SHORT = (9, 10)                            # short axes of the thin slabs: tuned in both precisions, and 9 * 10 lines / 10 columns
                                           # are not a multiple of any C > 2, so every pass with C > 2 has a ragged last tile


def lengths(prec):
    return sorted(e[0] for e in ENTRIES if e[1] == prec)


def entry_id(entry):
    return "%d%s" % (entry[0], "f64" if entry[1] == DOUBLE else "f32")


def thin_shape(n, axis, short=SHORT):
    """a slab whose transform length along `axis` (0 = X, 1 = Y, 2 = Z) is n and whose other two axes are `short`"""
    a, b = short
    return {2: (a, b, n), 1: (a, n, b), 0: (n, a, b)}[axis]


def threads(entry, axis):
    """threads per CTA of the entry's pass along `axis`: N / R * C"""
    k = {2: 0, 1: 1, 0: 2}[axis]
    return entry[0] // entry[3][k] * entry[2][k]
