"""CPU tests of the R2C / C2R slab schedules (dfft_plan_r2c_3d) without a GPU.

DRY_RUN plans record the passes they would launch.  The interpreter of test_dry_run.py gives the complex passes their
meaning; the real Z passes ("Z_R2C", "Z_C2R") are interpreted here with numpy's rfft / irfft, their real-side maps in units
of real elements and the two lines of a pair `pair` elements apart.  Every symbolic buffer is viewed both as complex128 and
as float64, so a plan that put complex data where real data belongs, or read or wrote past a user buffer, shows up as a
wrong answer or a touched canary.  The kernels' own arithmetic (two real lines per complex transform) is checked on the GPU
by test_gpu_r2c.py.

Also here: the fixed C2C schedules recorded before R2C existed (tests/golden/c2c_plan_ops.json) must come out unchanged,
and every unsupported R2C request must be refused with its error code."""
import json
import os

import numpy as np
import pytest

import distributedfft_b200 as dfft
from oracle import SlabGeometry
from test_dry_run import BUF1, IN, OUT, Machine, fake, run_alltoall, run_pass

HERE = os.path.dirname(os.path.abspath(__file__))
CANARY = 7.25e33


def real_view(m, addr, real):
    dev, b, byte_off = (addr >> 44) - 1, (addr >> 40) & 0xF, addr & ((1 << 40) - 1)
    arr = m.buf(dev, b)
    return (arr.view(np.float64), byte_off // 8) if real else (arr, byte_off // 16)


def run_real(m, op):
    """one real Z pass: tile t, pair c, line h of the pair at base + t*SB + c*cs + h*pair + e*es on each side"""
    fwd = op["op"] == "Z_R2C"
    N, H, C = op["N"], op["nzh"], op["C"]
    _, SBi, csi, esi = op["ia"]
    _, SBo, cso, eso = op["oa"]
    ldi, ldo = op["pair"]
    src, soff = real_view(m, op["in"], fwd)
    dst, doff = real_view(m, op["out"], not fwd)
    ei, eo = np.arange(N if fwd else H), np.arange(H if fwd else N)
    staged = []
    for tile in range(op["ntiles"]):
        for c in range(C):
            for h in range(2):
                if 2 * (tile * C + c) + h >= op["W"]:
                    continue
                v = src[soff + tile * SBi + c * csi + h * ldi + ei * esi]
                x = np.fft.rfft(v) if fwd else np.fft.irfft(v, n=N) * N
                if op["do_scale"]:
                    x = x * op["scale"]
                staged.append((tile, c, h, x))
    for tile, c, h, x in staged:
        dst[doff + tile * SBo + c * cso + h * ldo + eo * eso] = x


def simulate(n0, n1, n2, P, direction, inputs, flags):
    """inputs[d]: real x-slab (forward) or complex half-spectrum y-slab (backward) of device d"""
    H = n2 // 2 + 1
    m = Machine(SlabGeometry(n0, n1, H, P))
    plans, counts = [], []
    for d in range(P):
        rc, cc = dfft.local_size_r2c_3d(n0, n1, n2, P, d)
        counts.append((rc, cc))
        b1 = m.buf(d, BUF1)
        b1[:] = np.nan                                           # a read past the input slab poisons the result
        (b1.view(np.float64) if direction == dfft.FORWARD else b1)[: inputs[d].size] = inputs[d]
        m.buf(d, OUT).view(np.float64)[:] = CANARY               # a write past the output slab stays visible
        m.buf(d, IN).view(np.float64)[:] = CANARY                # the user's input is only copied at plan creation
        p = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, fake(d, IN), fake(d, OUT), None, d, P, direction, dfft.DOUBLE, flags | dfft.DRY_RUN)
        assert (p.in_count, p.out_count) == ((rc, cc) if direction == dfft.FORWARD else (cc, rc))
        assert not p.fused and p.pipeline_parts == 0
        plans.append(p)
    ops = []
    for p in plans:
        p.execute()
        ops.append(p.recorded_ops())
    for phase in (0, 1):
        for d in range(P):
            for op in ops[d]:
                if op["phase"] != phase or op["op"] == "alltoall":
                    continue
                run_real(m, op) if op["op"] in ("Z_R2C", "Z_C2R") else run_pass(m, op)
        if phase == 0:
            for d in range(P):
                for op in ops[d]:
                    if op["op"] == "alltoall":
                        run_alltoall(m, d, op)
    res = []
    for d in range(P):
        rc, cc = counts[d]
        out = m.buf(d, OUT)
        reals_used = 2 * cc if direction == dfft.FORWARD else rc
        res.append(out[:cc].copy() if direction == dfft.FORWARD else out.view(np.float64)[:rc].copy())
        assert np.all(out.view(np.float64)[reals_used:] == CANARY), (d, "write past the output slab")
        assert np.all(m.buf(d, IN).view(np.float64) == CANARY), (d, "the user's input buffer was touched")
    names = [[op["op"] for op in o] for o in ops]
    for p in plans:
        p.destroy()
    return res, names, ops


def y_slabs(S, P):
    """[x][y][nzh] -> per device q: [y_l][nzh][x] (the transposed spectrum layout)"""
    n1 = S.shape[1]
    yd = -(-n1 // P)
    return [S[:, q * yd: min(n1, (q + 1) * yd), :].transpose(1, 2, 0).reshape(-1) for q in range(P)]


def x_slabs(A, P):
    n0 = A.shape[0]
    xd = -(-n0 // P)
    return [A[q * xd: min(n0, (q + 1) * xd)].reshape(-1) for q in range(P)]


# P, n0, n1, n2: even and odd z lengths (9, 125, 243 odd), even and uneven splits, odd local line counts (n0_l * n1)
SHAPES = [(1, 5, 7, 9), (1, 6, 8, 10), (1, 4, 6, 125), (1, 3, 5, 16), (2, 5, 7, 9), (2, 8, 6, 12), (3, 7, 9, 16), (3, 10, 16, 9),
          (4, 10, 10, 8), (4, 8, 12, 243), (8, 24, 16, 10), (8, 30, 22, 9)]


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("P,n0,n1,n2", SHAPES)
def test_r2c_and_c2r_schedules_match_numpy(mode, P, n0, n1, n2):
    flags = dfft.EXCHANGE_P2P if mode == "p2p" else dfft.EXCHANGE_NCCL
    rng = np.random.default_rng(P * 1000 + n0 * 100 + n1 * 10 + n2)
    H = n2 // 2 + 1
    A = rng.standard_normal((n0, n1, n2))
    ref = np.fft.rfftn(A)
    got, names, _ = simulate(n0, n1, n2, P, dfft.FORWARD, x_slabs(A, P), flags)
    assert names[0][0] == "Z_R2C"
    scale = np.abs(ref).max()
    for d, r in enumerate(y_slabs(ref, P)):
        assert np.abs(got[d] - r).max() <= 1e-12 * scale, (d, names[d])
    # C2R of a NON-Hermitian spectrum: what numpy.fft.irfftn returns, times N (imaginary parts at z = 0 and n2/2 ignored)
    S = rng.standard_normal((n0, n1, H)) + 1j * rng.standard_normal((n0, n1, H))
    bref = np.fft.irfftn(S, s=(n0, n1, n2), axes=(0, 1, 2)) * (n0 * n1 * n2)
    for flg, want in ((flags, bref), (flags | dfft.SCALE_BACKWARD, bref / (n0 * n1 * n2))):
        got, names, _ = simulate(n0, n1, n2, P, dfft.BACKWARD, y_slabs(S, P), flg)
        assert names[0][-1] == "Z_C2R"
        for d, r in enumerate(x_slabs(want, P)):
            assert np.abs(got[d] - r).max() <= 1e-12 * np.abs(want).max(), (d, flg, names[d])


@pytest.mark.parametrize("n0,n1,n2", [(5, 7, 9), (6, 8, 10), (4, 12, 16)])
def test_natural_spectrum(n0, n1, n2):
    rng = np.random.default_rng(n2)
    A = rng.standard_normal((n0, n1, n2))
    ref = np.fft.rfftn(A)
    got, names, _ = simulate(n0, n1, n2, 1, dfft.FORWARD, [A.reshape(-1)], dfft.NATURAL_SPECTRUM)
    assert np.abs(got[0] - ref.reshape(-1)).max() <= 1e-12 * np.abs(ref).max()
    S = rng.standard_normal(ref.shape) + 1j * rng.standard_normal(ref.shape)
    back, _, _ = simulate(n0, n1, n2, 1, dfft.BACKWARD, [S.reshape(-1)], dfft.NATURAL_SPECTRUM | dfft.SCALE_BACKWARD)
    assert np.abs(back[0] - np.fft.irfftn(S, s=(n0, n1, n2), axes=(0, 1, 2)).reshape(-1)).max() <= 1e-12 * np.abs(S).max()


def test_fusion_and_pipeline_flags_have_no_effect(monkeypatch):
    """the real Z pass has no fused or pipelined form: the flags and their environment variables are accepted and change nothing"""
    n0, n1, n2 = 16, 16, 16
    for P, base in ((1, 0), (4, dfft.EXCHANGE_P2P)):
        def ops(flags):
            p = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, fake(0, IN), fake(0, OUT), None, 0, P, dfft.FORWARD, dfft.DOUBLE, base | flags | dfft.DRY_RUN)
            p.execute()
            out = (p.recorded_ops(), p.fused, p.pipeline_parts)
            p.destroy()
            return out
        plain = ops(0)
        for flags in (dfft.FORCE_FUSE, dfft.OVERLAP_X, dfft.FORCE_PIPELINE, dfft.FORCE_FUSE | dfft.OVERLAP_X | dfft.FORCE_PIPELINE):
            assert ops(flags) == plain
        for var, val in (("DFFT_FUSE", "1"), ("DFFT_OVERLAP", "1"), ("DFFT_PIPELINE", "1")):
            monkeypatch.setenv(var, val)
            assert ops(0) == plain
            monkeypatch.delenv(var)
        assert plain[1:] == (False, 0)


def test_unsupported_requests_are_refused():
    def code(n0, n1, n2, inp, out, flags=0, P=1, prec=dfft.DOUBLE, direction=dfft.FORWARD):
        try:
            p = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, inp, out, None, 0, P, direction, prec, flags | dfft.DRY_RUN)
        except dfft.DfftError as e:
            return int(str(e).split("(")[1].split(")")[0]), str(e)
        p.destroy()
        return 0, ""
    i, o = fake(0, IN), fake(0, OUT)
    assert code(8, 8, 16, i, o)[0] == 0
    assert code(8, 8, 16, i, None)[0] == -1                                   # in place (NULL out)
    assert code(8, 8, 16, i, i)[0] == -1                                      # in place (out == in)
    rc, msg = code(8, 8, 16, i, o, dfft.EXCHANGE_STAGED)
    assert rc == -3 and "STAGED" in msg
    assert code(8, 8, 16, i, o, dfft.EXCHANGE_STAGED, P=2)[0] == -3
    assert dfft.length_kind(14) == 1
    rc, msg = code(8, 8, 14, i, o)                                            # generic z length: no tuned kernel
    assert rc == -3 and "tuned" in msg
    assert code(8, 8, 17, i, o)[0] == -3                                      # unsupported length
    assert code(14, 14, 16, i, o)[0] == 0                                     # y and x may be any C2C length
    assert code(8, 8, 16, i, o + 8)[0] == -1                                  # misaligned fp64 complex output
    assert code(8, 8, 16, i + 8, o, direction=dfft.BACKWARD)[0] == -1         # misaligned fp64 complex input
    assert code(8, 8, 16, i + 8, o)[0] == 0                                   # a real fp64 buffer needs 8 bytes
    assert code(8, 8, 16, i + 4, o)[0] == -1
    assert code(8, 8, 16, i, o + 8, prec=dfft.FLOAT)[0] == 0                  # fp32: accepted (register-staged kernels only)
    p = dfft.fft_mpi_plan_dft_r2c_3d(8, 8, 16, i, o, None, 0, 1, dfft.FORWARD, dfft.DOUBLE, dfft.DRY_RUN)
    with pytest.raises(dfft.DfftError, match=r"\(-3\)"):
        p.execute_stage(0)
    p.destroy()


def test_local_sizes():
    for P, n0, n1, n2 in SHAPES:
        g = SlabGeometry(n0, n1, n2 // 2 + 1, P)
        for d in range(P):
            assert dfft.local_size_r2c_3d(n0, n1, n2, P, d) == (g.n0l(d) * n1 * n2, n0 * g.n1l(d) * (n2 // 2 + 1))
    with pytest.raises(dfft.DfftError):
        dfft.local_size_r2c_3d(8, 8, 8, 2, 2)


# ---- the C2C schedules are unchanged ------------------------------------------------------------------------------------
def _golden():
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_c2c_plan_ops as mk
    return mk


def test_c2c_schedules_are_unchanged(monkeypatch):
    mk = _golden()
    for v in mk.SCHEDULE_ENV:
        monkeypatch.delenv(v, raising=False)
    with open(os.path.join(HERE, "golden", "c2c_plan_ops.json")) as f:
        want = json.load(f)
    assert len(want) == 2 * len(mk.CASES)
    for P, n0, n1, n2, flags in mk.CASES:
        for direction in (dfft.FORWARD, dfft.BACKWARD):
            k = mk.key(P, n0, n1, n2, flags, direction)
            assert mk.record(P, n0, n1, n2, flags, direction) == want[k], k
