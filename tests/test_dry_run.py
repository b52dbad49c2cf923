"""CPU tests of the whole multi-device schedule without a GPU.

A DFFT_DRY_RUN plan makes no CUDA call: its buffers are symbolic addresses and dfft_execute records the passes it
would launch (affine maps, chunk tables, peer bases, scale / inverse / twiddle flags).  The interpreter below gives
those records their meaning -- "for every tile and column: gather N points through the input map, transform,
scatter through the output map", which is exactly what fft_tile_kernel / fft_fused*_kernel do on the device (the
kernels themselves are checked against the oracle on the GPU) -- on numpy arrays standing in for every device's
buffers, and the result is compared with the CPU oracle's restatement of the reference stages
(3dmpifft_opt/include/fft_mpi_3d_api.cpp:181-214).  This pins the host logic: slab geometry, pack/unpack chunk
tables, exchange offsets, uneven splits, fused / single-kernel / natural-order variants."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from oracle import BACKWARD, FORWARD, COracle, NumpySlab, SlabGeometry

ESZ = 16
BUF1, OUT, WORK, MID, IN = 1, 2, 3, 4, 5


def fake(dev, buf):
    return ((dev + 1) << 44) | (buf << 40)


def decode(addr):
    return (addr >> 44) - 1, (addr >> 40) & 0xF, (addr & ((1 << 40) - 1)) // ESZ


class Machine:
    def __init__(self, g):
        self.g = g
        self.mem = {}

    def buf(self, dev, b):
        key = (dev, b)
        if key not in self.mem:
            self.mem[key] = np.zeros(self.g.max_count(dev) + 64, dtype=np.complex128)
        return self.mem[key]

    def view(self, addr):
        dev, b, off = decode(addr)
        return self.buf(dev, b), off


def run_pass(m, op):
    N, C, G, W = op["N"], op["C"], op["G"], op["W"]
    SAi, SBi, csi, esi = op["ia"]
    SAo, SBo, cso, eso = op["oa"]
    e = np.arange(N)
    staged = []
    for tile in range(op["ntiles"]):
        a, b = divmod(tile, G)
        for c in range(C):
            if b * C + c >= W:
                continue
            if "ci" in op:
                ci = op["ci"]
                q = np.minimum(e // ci["ediv"], ci["nchunks"] - 1)
                v = np.empty(N, dtype=np.complex128)
                for qq in range(ci["nchunks"]):
                    sel = q == qq
                    if sel.any():
                        arr, off = m.view(ci["cptr"][qq])
                        v[sel] = arr[off + a * ci["SAq"][qq] + b * SBi + c * csi + (e[sel] - qq * ci["ediv"]) * esi]
            else:
                arr, off = m.view(op["in"])
                v = arr[off + a * SAi + b * SBi + c * csi + e * esi]
            x = np.fft.ifft(v) * N if op["inv"] else np.fft.fft(v)
            if op["tw_n"]:
                w = np.exp(-2j * np.pi * (((b * C + c) * e) % op["tw_n"]) / op["tw_n"])
                x = x * (np.conj(w) if op["inv"] else w)
            if op["do_scale"]:
                x = x * op["scale"]
            staged.append((a, b, c, x))
    # all loads of a pass happen-before its stores only per tile on the device; in-place passes touch disjoint tiles,
    # so storing after the loop is equivalent and keeps the interpreter simple
    for a, b, c, x in staged:
        if "co" in op:
            co = op["co"]
            q = np.minimum(e // co["ediv"], co["nchunks"] - 1)
            for qq in range(co["nchunks"]):
                sel = q == qq
                if sel.any():
                    arr, off = m.view(co["cptr"][qq])
                    arr[off + a * co["SAq"][qq] + b * SBo + c * cso + (e[sel] - qq * co["ediv"]) * eso] = x[sel]
        else:
            arr, off = m.view(op["out"])
            arr[off + a * SAo + b * SBo + c * cso + e * eso] = x


def run_alltoall(m, dev, op):
    src, soff = m.view(op["send"])
    for q, so, ro, cnt in op["chunks"]:
        rdev, rbuf, roff0 = decode(op["recv"])
        dst = m.buf(q, rbuf)          # the same buffer on the receiving device
        dst[roff0 + ro: roff0 + ro + cnt] = src[soff + so: soff + so + cnt]


def schedule(ops, nphases=2):
    """(device, record) in the order the interpreters run them: per phase, the passes of every device, then the phase's
    all-to-alls (C2C plans record two phases, convolve plans four)"""
    for phase in range(nphases):
        for a2a in (False, True):
            for d, o in enumerate(ops):
                for op in o:
                    if op["phase"] == phase and (op["op"] == "alltoall") == a2a:
                        yield d, op


def dry_ops(n0, n1, n2, P, direction, flags, precision=dfft.DOUBLE, inplace=False):
    """the records of one execute of each of the P per-device DRY_RUN C2C plans, and whether each plan fuses its t0"""
    plans = [dfft.fft_mpi_plan_dft_c2c_3d(n0, n1, n2, fake(d, IN), None if inplace else fake(d, OUT), None, d, P, direction, precision,
                                          flags | dfft.DRY_RUN) for d in range(P)]
    ops = []
    for p in plans:
        p.execute()
        ops.append(p.recorded_ops())
    fused = [p.fused for p in plans]
    for p in plans:
        p.destroy()
    return ops, fused


def simulate(n0, n1, n2, P, direction, inputs, flags, inplace=False):
    g = SlabGeometry(n0, n1, n2, P)
    m = Machine(g)
    for d in range(P):
        m.buf(d, BUF1)[: inputs[d].size] = inputs[d]      # the plan snapshots `in` into bufferDev1 (api.cpp:76-77)
    ops, fused = dry_ops(n0, n1, n2, P, direction, flags, inplace=inplace)
    for d, op in schedule(ops):
        if op["op"] == "alltoall":
            run_alltoall(m, d, op)
        else:
            run_pass(m, op)
    outb = IN if inplace else OUT
    res = [m.buf(d, outb)[: g.max_count(d)].copy() for d in range(P)]
    names = [[op["op"] for op in o] for o in ops]
    return res, names, fused


@pytest.fixture(scope="module")
def co():
    return COracle()


def oracle(co, g, A, direction):
    ns = NumpySlab(g.n0, g.n1, g.n2, g.P)
    if direction == FORWARD:
        b1 = ns.scatter_input(A)
    else:
        b1 = []
        for q in range(g.P):
            b = np.zeros(g.max_count(q), dtype=np.complex128)
            blk = A[:, q * g.yd: q * g.yd + g.n1l(q), :].transpose(1, 2, 0).reshape(-1)
            b[: blk.size] = blk
            b1.append(b)
    inputs = [b.copy() for b in b1]
    b2 = [np.zeros_like(b) for b in b1]
    co.slab_execute(g, b1, b2, direction)
    return inputs, b2


SHAPES = [(1, 8, 16, 4), (1, 12, 10, 24), (2, 16, 16, 16), (2, 10, 9, 4), (3, 10, 9, 4), (3, 9, 10, 4), (4, 12, 10, 10), (4, 16, 8, 8),
          (8, 24, 16, 16), (3, 15, 22, 26)]


@pytest.mark.parametrize("mode", ["p2p", "p2p-nofuse", "nccl"])
@pytest.mark.parametrize("P,n0,n1,n2", SHAPES)
def test_recorded_schedule_reproduces_the_reference_stages(co, mode, P, n0, n1, n2):
    flags = {"p2p": dfft.EXCHANGE_P2P, "p2p-nofuse": dfft.EXCHANGE_P2P | dfft.NO_FUSE, "nccl": dfft.EXCHANGE_NCCL}[mode]
    g = SlabGeometry(n0, n1, n2, P)
    rng = np.random.default_rng(n0 * 100 + n1 * 10 + P)
    A = rng.standard_normal((n0, n1, n2)) + 1j * rng.standard_normal((n0, n1, n2))
    for direction in (FORWARD, BACKWARD):
        inputs, ref = oracle(co, g, A, direction)
        got, names, fused = simulate(n0, n1, n2, P, direction, inputs, flags)
        scale = max(np.abs(r).max() for r in ref)
        for d in range(P):
            n = g.out_count(d) if direction == FORWARD else g.in_count(d)
            assert np.abs(got[d][:n] - ref[d][:n]).max() <= 1e-11 * scale, (mode, direction, d, names[d])
        if mode == "p2p" and P > 1 and n1 == n2 and dfft.length_kind(n1) == 2:
            assert all(fused) and any(nm.startswith("fused") for nm in names[0])
        if mode != "p2p":
            assert not any(fused)


@pytest.mark.parametrize("P,n", [(2, 64), (4, 64), (8, 64)])
def test_single_kernel_forward_schedule(co, P, n):
    """DFFT_OVERLAP_X: the three roles of fft_fused3_kernel (Z -> own intermediate, Y -> peers' receive buffers, X from the
    receive buffer) reproduce the reference's forward result."""
    g = SlabGeometry(n, n, n, P)
    rng = np.random.default_rng(P)
    A = rng.standard_normal((n, n, n)) + 1j * rng.standard_normal((n, n, n))
    inputs, ref = oracle(co, g, A, FORWARD)
    got, names, fused = simulate(n, n, n, P, FORWARD, inputs, dfft.EXCHANGE_P2P | dfft.OVERLAP_X)
    assert names[0] == ["ovlZ", "ovlY", "ovlX"]
    scale = max(np.abs(r).max() for r in ref)
    for d in range(P):
        assert np.abs(got[d][: g.out_count(d)] - ref[d][: g.out_count(d)]).max() <= 1e-11 * scale


PIPE_SHAPES = [("p2p", 4, 64, 64, 64, "2"), ("p2p", 8, 64, 64, 64, "4"), ("p2p", 2, 8, 128, 128, None), ("p2p", 4, 8, 12, 128, None), ("p2p", 3, 10, 9, 128, None), ("p2p", 8, 16, 64, 64, "2"),
               ("p2p", 2, 6, 64, 64, "1"), ("nccl", 2, 8, 16, 128, None), ("nccl", 4, 8, 8, 64, "2"), ("nccl", 8, 64, 64, 64, "4")]


@pytest.mark.parametrize("mode,P,n0,n1,n2,parts", PIPE_SHAPES)
def test_stream_pipelined_forward_schedule(co, monkeypatch, mode, P, n0, n1, n2, parts):
    """The z-part pipeline (fwd_pipelined): Z, Y parts with part-major peer stores / packed send parts + per-part
    all-to-all, X parts reading the part-major receive buffer -- reproduces the reference's forward result for even
    and uneven splits, fused (square planes) and two-sweep t0, P2P and NCCL exchanges."""
    if parts:
        monkeypatch.setenv("DFFT_PARTS", parts)
    g = SlabGeometry(n0, n1, n2, P)
    rng = np.random.default_rng(P + n2)
    A = rng.standard_normal((n0, n1, n2)) + 1j * rng.standard_normal((n0, n1, n2))
    inputs, ref = oracle(co, g, A, FORWARD)
    flags = (dfft.EXCHANGE_P2P if mode == "p2p" else dfft.EXCHANGE_NCCL) | dfft.FORCE_PIPELINE
    got, names, fused = simulate(n0, n1, n2, P, FORWARD, inputs, flags)
    K = int(parts) if parts else 4
    if mode == "p2p" and n0 == n1 == n2:
        # cubes: chain of two-role kernels on one stream ([Z + Y0] [Y1 + X0] ... [X K-1]), fft_fused_yx_kernel
        assert names[0] == ["fusedZ", "fusedY"] + ["Y_CO", "XF"] * (K - 1) + ["XF"], names[0]
    for d in range(P):
        assert names[d].count("XF") == K, names[d]
        if mode == "nccl":
            assert names[d].count("alltoall") == K and names[d][0] == "Z"
        elif n1 == n2 and dfft.length_kind(n1) == 2:
            assert names[d][:2] == ["fusedZ", "fusedY"] and names[d].count("Y_CO") == K - 1
        else:
            assert names[d][0] == "Z" and names[d].count("Y_CO") == K
    scale = max(np.abs(r).max() for r in ref)
    for d in range(P):
        assert np.abs(got[d][: g.out_count(d)] - ref[d][: g.out_count(d)]).max() <= 1e-11 * scale, d
    # backward: inverse X parts (chunked to the destinations' part-major receive buffers), inverse Y parts (chunked load), the
    # last one fused with the inverse Z pass when the planes are square
    binputs, bref = oracle(co, g, A, BACKWARD)
    bgot, bnames, _ = simulate(n0, n1, n2, P, BACKWARD, binputs, flags)
    bscale = max(np.abs(r).max() for r in bref)
    for d in range(P):
        assert bnames[d].count("XB_CO") == K, bnames[d]
        if mode == "nccl":
            assert bnames[d].count("alltoall") == K
        assert np.abs(bgot[d][: g.in_count(d)] - bref[d][: g.in_count(d)]).max() <= 1e-11 * bscale, (d, bnames[d])
    # DFFT_NO_PIPELINE falls back to the single-part schedule
    got2, names2, _ = simulate(n0, n1, n2, P, FORWARD, inputs, (flags & ~dfft.FORCE_PIPELINE) | dfft.NO_PIPELINE)
    assert names2[0].count("XF") == 1
    for d in range(P):
        assert np.abs(got2[d][: g.out_count(d)] - ref[d][: g.out_count(d)]).max() <= 1e-11 * scale, d


@pytest.mark.parametrize("n0,n1,n2", [(8, 16, 4), (12, 10, 24), (15, 22, 26)])
def test_natural_spectrum_schedule(n0, n1, n2):
    rng = np.random.default_rng(n0)
    A = rng.standard_normal((n0, n1, n2)) + 1j * rng.standard_normal((n0, n1, n2))
    ref = np.fft.fftn(A).reshape(-1)
    got, names, _ = simulate(n0, n1, n2, 1, FORWARD, [A.reshape(-1)], dfft.NATURAL_SPECTRUM)
    assert np.abs(got[0][: ref.size] - ref).max() <= 1e-11 * np.abs(ref).max()
    back, _, _ = simulate(n0, n1, n2, 1, BACKWARD, [ref], dfft.NATURAL_SPECTRUM)
    assert np.abs(back[0][: ref.size] / A.size - A.reshape(-1)).max() <= 1e-11


def test_in_place_and_scale_schedule():
    n0, n1, n2 = 8, 16, 4
    rng = np.random.default_rng(1)
    A = rng.standard_normal((n0, n1, n2)) + 1j * rng.standard_normal((n0, n1, n2))
    ref = np.fft.fftn(A).transpose(1, 2, 0).reshape(-1)
    got, _, _ = simulate(n0, n1, n2, 1, FORWARD, [A.reshape(-1)], 0, inplace=True)
    assert np.abs(got[0][: ref.size] - ref).max() <= 1e-11 * np.abs(ref).max()
    back, _, _ = simulate(n0, n1, n2, 1, BACKWARD, [ref], dfft.SCALE_BACKWARD)
    assert np.abs(back[0][: ref.size] - A.reshape(-1)).max() <= 1e-11


class FlatMachine:
    """one device, flat buffers of arbitrary size (lines plans)"""

    def __init__(self, size):
        self.mem = {}
        self.size = size

    def view(self, addr):
        dev, b, off = decode(addr)
        if b not in self.mem:
            self.mem[b] = np.zeros(self.size, dtype=np.complex128)
        return self.mem[b], off


@pytest.mark.parametrize("n", [8192, 16384, 6561, 12000, 16807, 15625, 131072])
def test_four_step_long_line_schedule(n):
    """Lines beyond one shared-memory line: the two recorded passes (FFT along n1 + twiddle + transposed store, then the
    strided FFT along n2) give the natural-order transform, forward and inverse."""
    lines = 2
    rng = np.random.default_rng(n)
    x = rng.standard_normal((lines, n)) + 1j * rng.standard_normal((lines, n))
    for direction in (FORWARD, BACKWARD):
        ops = dfft.lines_ops(n, 1, lines, lines, n, 0, direction)
        assert [o["op"] for o in ops] == ["XF_TW", "Y"] and ops[0]["tw_n"] == n and ops[0]["N"] * ops[1]["N"] == n
        m = FlatMachine(lines * n)
        m.view(fake(0, BUF1))[0][:] = x.reshape(-1)
        for op in ops:
            run_pass(m, op)
        ref = np.fft.fft(x, axis=1) if direction == FORWARD else np.fft.ifft(x, axis=1) * n
        got = m.view(fake(0, BUF1))[0].reshape(lines, n)
        assert np.abs(got - ref).max() <= 1e-10 * np.abs(ref).max(), (n, direction)


def test_lines_plan_schedules_1d_and_2d():
    rng = np.random.default_rng(5)
    # strided columns of 3 row-major matrices (n rows x 21 columns), and a batched 2-D plan
    n, cols, mats = 96, 21, 3
    b = rng.standard_normal((mats, n, cols)) + 1j * rng.standard_normal((mats, n, cols))
    ops = dfft.lines_ops(n, cols, mats * cols, cols, 1, n * cols, FORWARD)
    m = FlatMachine(b.size)
    m.view(fake(0, BUF1))[0][:] = b.reshape(-1)
    for op in ops:
        run_pass(m, op)
    assert np.abs(m.view(fake(0, BUF1))[0].reshape(b.shape) - np.fft.fft(b, axis=1)).max() <= 1e-11 * n
    nx, ny, batch = 64, 48, 3
    a = rng.standard_normal((batch, ny, nx)) + 1j * rng.standard_normal((batch, ny, nx))
    for direction in (FORWARD, BACKWARD):
        ops = dfft.lines_ops(nx, ny, batch, 0, 0, 0, direction, two_d=True)
        m = FlatMachine(a.size)
        m.view(fake(0, BUF1))[0][:] = a.reshape(-1)
        for op in ops:
            run_pass(m, op)
        ref = np.fft.fft2(a, axes=(1, 2)) if direction == FORWARD else np.fft.ifft2(a, axes=(1, 2)) * nx * ny
        assert np.abs(m.view(fake(0, BUF1))[0].reshape(a.shape) - ref).max() <= 1e-11 * np.abs(ref).max()


def test_lines_plans_take_at_most_2_31_minus_1_rows():
    """A pass's row (or column) count is a 32-bit kernel argument: 1-D and 2-D plans with more are DFFT_EUNSUPPORTED, as the
    3-D, real and convolve plans are, rather than transforming only the rows below the limit."""
    rows = 1 << 31
    ops = dfft.lines_ops(2, 1, rows - 1, rows - 1, 2, 0, FORWARD)
    assert [(o["op"], o["W"]) for o in ops] == [("Z", rows - 1)]
    for args, two_d in (((2, 1, rows, rows, 2, 0), False),            # contiguous lines
                        ((2, rows, rows, rows, 1, 0), False),         # strided columns
                        ((65536, 1, rows, rows, 65536, 0), False),    # four-step long lines
                        ((2, 2, rows >> 1, 0, 0, 0), True),           # 2-D: ny * batch rows
                        ((16, 16, 1 << 60, 0, 0, 0), True)):          # 2-D: ny * batch beyond 64 bits
        with pytest.raises(dfft.DfftError, match=r"\(-3\)"):
            dfft.lines_ops(*args, FORWARD, two_d=two_d)


def test_random_geometries_all_exchanges(co):
    """Seeded random sweep over device counts, tuned and generic lengths, even and uneven splits, both directions."""
    rng = np.random.default_rng(2026)
    lengths = [4, 6, 8, 9, 10, 12, 16, 24, 5, 7, 14, 15, 20, 21, 22, 26, 27, 28, 30, 32]
    done = 0
    while done < 24:
        P = int(rng.integers(1, 7))
        n0, n1, n2 = (int(x) for x in rng.choice(lengths, 3))
        g = SlabGeometry(n0, n1, n2, P)
        if g.last_n0 < 1 or g.last_n1 < 1:
            continue
        flags = [dfft.EXCHANGE_P2P, dfft.EXCHANGE_NCCL, dfft.EXCHANGE_P2P | dfft.NO_FUSE][done % 3]
        direction = FORWARD if done % 2 == 0 else BACKWARD
        A = rng.standard_normal((n0, n1, n2)) + 1j * rng.standard_normal((n0, n1, n2))
        inputs, ref = oracle(co, g, A, direction)
        got, names, _ = simulate(n0, n1, n2, P, direction, inputs, flags)
        scale = max(np.abs(r).max() for r in ref)
        for d in range(P):
            n = g.out_count(d) if direction == FORWARD else g.in_count(d)
            assert np.abs(got[d][:n] - ref[d][:n]).max() <= 1e-11 * scale, (P, n0, n1, n2, flags, direction, d, names[d])
        done += 1


def test_random_geometries_pipelined_schedules(co, monkeypatch):
    """Seeded random sweep with DFFT_FORCE_PIPELINE: z axes long enough to be cut into parts, x / y extents even and uneven over
    1..8 devices, P2P and NCCL, both directions, 2 or 4 parts, chain (cubes) and two-stream schedules.  Where a geometry does not
    meet a pipeline's preconditions the plan falls back to the plain schedule -- the result must be right either way."""
    rng = np.random.default_rng(77)
    done = piped = 0
    while done < 20:
        P = int(rng.integers(2, 9))
        n2 = int(rng.choice([64, 128]))
        cube = done % 5 == 0
        n0, n1 = (n2, n2) if cube else (int(x) for x in rng.choice([8, 9, 10, 12, 16, 20, 24, 30, 32, 64], 2))
        g = SlabGeometry(n0, n1, n2, P)
        if g.last_n0 < 1 or g.last_n1 < 1:
            continue
        nccl = done % 3 == 1
        direction = FORWARD if done % 2 == 0 else BACKWARD
        monkeypatch.setenv("DFFT_PARTS", "2" if done % 4 < 2 else "4")
        A = rng.standard_normal((n0, n1, n2)) + 1j * rng.standard_normal((n0, n1, n2))
        inputs, ref = oracle(co, g, A, direction)
        flags = (dfft.EXCHANGE_NCCL if nccl else dfft.EXCHANGE_P2P) | dfft.FORCE_PIPELINE
        got, names, _ = simulate(n0, n1, n2, P, direction, inputs, flags)
        scale = max(np.abs(r).max() for r in ref)
        for d in range(P):
            n = g.out_count(d) if direction == FORWARD else g.in_count(d)
            assert np.abs(got[d][:n] - ref[d][:n]).max() <= 1e-11 * scale, (P, n0, n1, n2, flags, direction, d, names[d])
        piped += len(names[0]) > 4
        done += 1
    assert piped >= 10, piped


def test_default_pipeline_policy(monkeypatch):
    """Which schedule a plan picks by default (dfft_plan_c2c_3d, measured policy of DESIGN.md 5.1): the kernel chain for cubes
    with axes >= 1024 points from 4 devices on (P2P), the plain schedule everywhere else; flags and environment override."""
    for var in ("DFFT_PIPELINE", "DFFT_PARTS", "DFFT_PIPE_MODE"):
        monkeypatch.delenv(var, raising=False)

    def plan(n0, n1, n2, P, flags=0, direction=FORWARD):
        p = dfft.fft_mpi_plan_dft_c2c_3d(n0, n1, n2, fake(0, IN), fake(0, OUT), None, 0, P, direction, dfft.DOUBLE, flags | dfft.DRY_RUN)
        out = (p.pipeline_parts, p.pipeline_chain)
        p.destroy()
        return out

    assert plan(1024, 1024, 1024, 4) == (4, True)
    assert plan(1024, 1024, 1024, 8) == (4, True)
    assert plan(1024, 1024, 1024, 2) == (0, False)                         # 2 devices: L2-fabric bound, nothing to hide
    assert plan(512, 512, 512, 8) == (0, False)                            # short X pass: a tie at 4 devices, not the default
    assert plan(768, 768, 768, 8) == (0, False)
    assert plan(1024, 1024, 1024, 4, dfft.EXCHANGE_NCCL) == (0, False)     # NCCL: opt-in
    assert plan(1024, 1024, 1024, 4, direction=BACKWARD) == (0, False)     # backward: opt-in (two-stream schedule)
    assert plan(1024, 1024, 1024, 4, dfft.NO_PIPELINE) == (0, False)
    assert plan(512, 512, 512, 2, dfft.FORCE_PIPELINE) == (4, True)
    assert plan(512, 512, 512, 4, dfft.EXCHANGE_NCCL | dfft.FORCE_PIPELINE) == (4, False)
    assert plan(512, 512, 512, 4, dfft.FORCE_PIPELINE, BACKWARD) == (4, False)
    assert plan(64, 512, 512, 4, dfft.FORCE_PIPELINE) == (4, False)        # not a cube: two streams
    assert plan(512, 512, 512, 1, dfft.FORCE_PIPELINE) == (0, False)
    monkeypatch.setenv("DFFT_PIPELINE", "1")
    assert plan(512, 512, 512, 4) == (4, True)
    monkeypatch.setenv("DFFT_PIPE_MODE", "streams")
    assert plan(512, 512, 512, 4) == (4, False)
    monkeypatch.setenv("DFFT_PIPELINE", "0")
    assert plan(1024, 1024, 1024, 8) == (0, False)
