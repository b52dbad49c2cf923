"""CPU tests of the spectral convolution plans (dfft_plan_convolve_c2c_3d / dfft_plan_convolve_r2c_3d) without a GPU.

DRY_RUN plans record the passes they would launch.  The complex passes are interpreted by test_dry_run.run_pass, the real Z
passes by test_r2c_dry_run.run_real; the fused X pass ("XCONV", "XCONV_CO") is interpreted here: for every column, numpy's FFT
along x, the product with the multiplier gathered through the same input map from the recorded "mult" address, the inverse
(unnormalised), then the store through the output map or the chunk table.  A convolve plan records four phases: 0 forward half,
1 fused X pass, 2 the backward exchange, 3 backward half; every device runs a phase before any device runs the next, and the
all-to-alls of a phase run after its passes.

bufferDev1 and the multiplier are NaN past their slabs, the output is NaN-filled with canaries past its end, and the user's
input is a canary block: a read past a slab, a missed store or a write past a buffer shows up as a wrong answer or a touched
canary.  The results are compared with numpy's ifftn(fftn(A) * M) * N and irfftn(rfftn(A) * M) * N.  Also here: the fp64 bound
of the GPU tests (twice the single-transform bound of ldfft) accepts numpy's convolution and rejects one whose forward half has
a stage of 40-bit twiddles."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
import ldfft
from oracle import SlabGeometry
from test_dry_run import BUF1, IN, OUT, Machine, decode, fake, run_alltoall, run_pass, schedule
from test_r2c_dry_run import run_real

CANARY = 7.25e33
MULT = 8


def run_conv(m, op):
    N, C, G, W = op["N"], op["C"], op["G"], op["W"]
    SAi, SBi, csi, esi = op["ia"]
    SAo, SBo, cso, eso = op["oa"]
    e = np.arange(N)
    src, soff = m.view(op["in"])
    mul, moff = m.view(op["mult"])
    staged = []
    for tile in range(op["ntiles"]):
        a, b = divmod(tile, G)
        for c in range(C):
            if b * C + c >= W:
                continue
            rel = a * SAi + b * SBi + c * csi + e * esi
            x = np.fft.ifft(np.fft.fft(src[soff + rel]) * mul[moff + rel]) * N
            if op["do_scale"]:
                x = x * op["scale"]
            staged.append((a, b, c, x))
    for a, b, c, x in staged:
        if "co" in op:
            co = op["co"]
            q = np.minimum(e // co["ediv"], co["nchunks"] - 1)
            for qq in range(co["nchunks"]):
                sel = q == qq
                arr, off = m.view(co["cptr"][qq])
                arr[off + a * co["SAq"][qq] + b * SBo + c * cso + (e[sel] - qq * co["ediv"]) * eso] = x[sel]
        else:
            arr, off = m.view(op["out"])
            arr[off + a * SAo + b * SBo + c * cso + e * eso] = x


def x_slabs(A, P):
    xd = -(-A.shape[0] // P)
    return [A[q * xd: min(A.shape[0], (q + 1) * xd)].reshape(-1) for q in range(P)]


def y_slabs(M, P):
    yd = -(-M.shape[1] // P)
    return [M[:, q * yd: min(M.shape[1], (q + 1) * yd), :].reshape(-1) for q in range(P)]


def written(op):
    """buffer addresses a record stores to"""
    if op["op"] == "alltoall":
        return [op["recv"]]
    return op["co"]["cptr"] if "co" in op else [op["out"]]


def simulate(n0, n1, n2, P, A, M, flags, real=False, inplace=False, mult_offset=0):
    H = n2 // 2 + 1 if real else n2
    g = SlabGeometry(n0, n1, H, P)
    m = Machine(g)
    plans, counts = [], []
    for d in range(P):
        cnt = g.n0l(d) * n1 * n2
        counts.append(cnt)
        b1 = m.buf(d, BUF1)
        b1[:] = np.nan
        (b1.view(np.float64) if real else b1)[:cnt] = x_slabs(A, P)[d]
        mb = m.buf(d, MULT)
        mb[:] = np.nan
        mslab = y_slabs(M, P)[d]
        mb[mult_offset: mult_offset + mslab.size] = mslab
        m.buf(d, IN).view(np.float64)[:] = CANARY
        m.buf(d, OUT).view(np.float64)[:] = CANARY
        outb = IN if inplace else OUT
        (m.buf(d, outb).view(np.float64) if real else m.buf(d, outb))[:cnt] = np.nan
        p = dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, fake(d, IN), None if inplace else fake(d, OUT), None, d, P, dfft.DOUBLE,
                                              flags | dfft.DRY_RUN, real=real)
        assert (p.in_count, p.out_count) == (cnt, cnt)
        plans.append(p)
    keep = {k: v.copy() for k, v in m.mem.items() if k[1] in (BUF1, MULT)}
    ops = []
    for d, p in enumerate(plans):
        p.execute_convolve(fake(d, MULT) + 16 * mult_offset)
        ops.append(p.recorded_ops())
    for d, op in schedule(ops, 4):
        if op["op"] == "alltoall":
            run_alltoall(m, d, op)
        elif op["op"].startswith("XCONV"):
            run_conv(m, op)
        elif op["op"] in ("Z_R2C", "Z_C2R"):
            run_real(m, op)
        else:
            run_pass(m, op)
    res = []
    for d in range(P):
        outbuf = m.buf(d, IN if inplace else OUT)
        flat = outbuf.view(np.float64) if real else outbuf
        res.append(flat[: counts[d]].copy())
        assert np.all(outbuf.view(np.float64)[(1 if real else 2) * counts[d]:] == CANARY), (d, "write past the output slab")
        if not inplace:
            assert np.all(m.buf(d, IN).view(np.float64) == CANARY), (d, "the user's input buffer was touched")
    for k, v in keep.items():
        assert np.array_equal(m.mem[k], v, equal_nan=True), (k, "bufferDev1 or the multiplier was written")
    for o in ops:
        for op in o:
            for addr in written(op):
                assert decode(addr)[1] not in (BUF1, MULT), op["op"]
    for p in plans:
        p.destroy()
    return res, [[op["op"] for op in o] for o in ops], ops


def reference(A, M, real, scaled):
    n = A.size
    if real:
        r = np.fft.irfftn(np.fft.rfftn(A) * M, s=A.shape, axes=(0, 1, 2))
    else:
        r = np.fft.ifftn(np.fft.fftn(A) * M)
    return r if scaled else r * n


def case(n0, n1, n2, real, seed):
    rng = np.random.default_rng(seed)
    H = n2 // 2 + 1 if real else n2
    A = rng.standard_normal((n0, n1, n2)) if real else rng.standard_normal((n0, n1, n2)) + 1j * rng.standard_normal((n0, n1, n2))
    M = rng.standard_normal((n0, n1, H)) + 1j * rng.standard_normal((n0, n1, H))
    return A, M


def check(n0, n1, n2, P, flags, real, inplace=False, seed=0, mult_offset=0):
    A, M = case(n0, n1, n2, real, seed + 1000 * P + n0)
    got, names, ops = simulate(n0, n1, n2, P, A, M, flags, real, inplace, mult_offset)
    want = x_slabs(reference(A, M, real, bool(flags & dfft.SCALE_BACKWARD)), P)
    scale = max(np.abs(w).max() for w in want)
    for d in range(P):
        assert np.abs(got[d] - want[d]).max() <= 1e-12 * scale, (d, names[d])
    return names, ops


SHAPES = [(1, 8, 16, 4), (1, 12, 10, 24), (1, 16, 16, 16), (2, 16, 16, 16), (2, 10, 9, 4), (3, 10, 12, 16), (3, 12, 10, 9),
          (4, 16, 8, 8), (4, 12, 10, 10), (8, 24, 16, 16), (8, 16, 16, 9)]


@pytest.mark.parametrize("real", [False, True], ids=["c2c", "r2c"])
@pytest.mark.parametrize("mode", ["p2p", "nccl", "p2p-nofuse", "p2p-forcefuse"])
@pytest.mark.parametrize("P,n0,n1,n2", SHAPES)
def test_convolve_schedules_match_numpy(P, n0, n1, n2, mode, real):
    flags = {"p2p": dfft.EXCHANGE_P2P, "nccl": dfft.EXCHANGE_NCCL, "p2p-nofuse": dfft.EXCHANGE_P2P | dfft.NO_FUSE,
             "p2p-forcefuse": dfft.EXCHANGE_P2P | dfft.FORCE_FUSE}[mode]
    names, _ = check(n0, n1, n2, P, flags, real)
    conv = [nm for nm in names[0] if nm.startswith("XCONV")]
    assert conv == (["XCONV_CO"] if P > 1 and mode != "nccl" else ["XCONV"]), names[0]
    assert not any(nm in ("XF", "XB", "XB_CO") for nm in names[0])
    if mode == "nccl" and P > 1:
        assert names[0].count("alltoall") == 2
    if real:
        assert names[0][0] == "Z_R2C" and names[0][-1] == "Z_C2R"


@pytest.mark.parametrize("real", [False, True], ids=["c2c", "r2c"])
@pytest.mark.parametrize("P,n0,n1,n2", [(1, 8, 6, 9), (1, 6, 8, 10), (2, 8, 12, 10), (3, 12, 10, 9), (4, 16, 8, 9)])
def test_scaled_in_place_and_odd_z(P, n0, n1, n2, real):
    for flags in (dfft.SCALE_BACKWARD, dfft.SCALE_BACKWARD | dfft.EXCHANGE_NCCL, 0):
        check(n0, n1, n2, P, flags, real, inplace=True, seed=flags)
        check(n0, n1, n2, P, flags, real, inplace=False, seed=flags + 1)


def test_multiplier_at_an_offset_is_read_through_its_own_base():
    check(8, 12, 10, 2, dfft.EXCHANGE_P2P, False, mult_offset=5)
    check(8, 12, 10, 1, 0, True, mult_offset=3)


def _phase_names(ops, phases):
    return [op["op"] for op in ops if op["phase"] in phases and op["op"] != "alltoall"]


@pytest.mark.parametrize("P,n", [(1, 16), (2, 16), (4, 16), (3, 12)])
@pytest.mark.parametrize("flags", [0, dfft.NO_FUSE, dfft.FORCE_FUSE, dfft.EXCHANGE_NCCL, dfft.EXCHANGE_NCCL | dfft.FORCE_FUSE])
def test_halves_select_t0_as_the_c2c_plans_do(P, n, flags):
    """the forward half runs the t0 kernels a C2C forward plan of the shape runs, the backward half those of a C2C backward plan"""
    flags |= dfft.EXCHANGE_P2P if not flags & dfft.EXCHANGE_NCCL else 0
    p = dfft.fft_mpi_plan_dft_convolve_3d(n, n, n, fake(0, IN), fake(0, OUT), None, 0, P, dfft.DOUBLE, flags | dfft.DRY_RUN)
    p.execute_convolve(fake(0, MULT))
    conv = p.recorded_ops()
    p.destroy()
    ref = {}
    for direction in (dfft.FORWARD, dfft.BACKWARD):
        q = dfft.fft_mpi_plan_dft_c2c_3d(n, n, n, fake(0, IN), fake(0, OUT), None, 0, P, direction, dfft.DOUBLE, flags | dfft.DRY_RUN)
        q.execute()
        ref[direction] = q.recorded_ops()
        q.destroy()
    assert _phase_names(conv, (0,)) == _phase_names(ref[dfft.FORWARD], (0,))
    assert _phase_names(conv, (3,)) == _phase_names(ref[dfft.BACKWARD], (1,))
    for op in conv:
        if op["phase"] in (0, 3) and op["op"] != "alltoall":
            assert op["inv"] == (1 if op["phase"] == 3 else 0), op


def test_pipeline_and_overlap_flags_have_no_effect(monkeypatch):
    for P, base in ((1, 0), (4, dfft.EXCHANGE_P2P), (4, dfft.EXCHANGE_NCCL)):
        def ops(flags):
            p = dfft.fft_mpi_plan_dft_convolve_3d(64, 64, 64, fake(0, IN), fake(0, OUT), None, 0, P, dfft.DOUBLE, base | flags | dfft.DRY_RUN)
            p.execute_convolve(fake(0, MULT))
            out = (p.recorded_ops(), p.pipeline_parts)
            p.destroy()
            return out
        plain = ops(0)
        for flags in (dfft.OVERLAP_X, dfft.FORCE_PIPELINE, dfft.NO_PIPELINE, dfft.OVERLAP_X | dfft.FORCE_PIPELINE):
            assert ops(flags) == plain
        for var in ("DFFT_OVERLAP", "DFFT_PIPELINE"):
            monkeypatch.setenv(var, "1")
            assert ops(0) == plain
            monkeypatch.delenv(var)
        assert plain[1] == 0


def _code(fn):
    try:
        fn()
    except dfft.DfftError as e:
        return int(str(e).split("(")[1].split(")")[0])
    return 0


def test_rejections(monkeypatch):
    i, o = fake(0, IN), fake(0, OUT)

    def mk(n0=16, n1=16, n2=16, flags=0, real=False, prec=dfft.DOUBLE, P=1, inp=i, out=o):
        return lambda: dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, inp, out, None, 0, P, prec, flags | dfft.DRY_RUN, real=real).destroy()
    for real in (False, True):
        assert _code(mk(real=real)) == 0
        assert _code(mk(real=real, out=None)) == 0 and _code(mk(real=real, out=i)) == 0          # in place
        assert _code(mk(real=real, flags=dfft.EXCHANGE_STAGED)) == -3
        assert _code(mk(real=real, flags=dfft.EXCHANGE_STAGED, P=2)) == -3
        assert dfft.length_kind(14) == 1
        assert _code(mk(n0=14, real=real)) == -3                                                 # generic x length
        assert _code(mk(n0=17, real=real)) == -3
        assert _code(mk(n1=17, real=real)) == -3                                                 # y length the C2C plan rejects
        assert _code(mk(n2=17, real=real)) == -3
        assert _code(mk(real=real, flags=dfft.NATURAL_SPECTRUM)) == -1
        assert _code(mk(real=real, flags=dfft.NATURAL_SPECTRUM, P=2)) == -1
    assert _code(mk(n2=14)) == 0                                                                 # generic z: fine for C2C ...
    assert _code(mk(n2=14, real=True)) == -3                                                     # ... not for the real z pass
    assert _code(mk(out=o + 8)) == -1                                                            # misaligned fp64 complex output
    assert _code(mk(out=o + 8, prec=dfft.FLOAT)) == 0
    assert _code(mk(out=o + 8, real=True)) == 0 and _code(mk(inp=i + 8, real=True)) == 0        # real fp64 buffers need 8 bytes
    assert _code(mk(out=o + 4, real=True)) == -1 and _code(mk(inp=i + 4, real=True)) == -1
    assert _code(mk(out=o + 4, real=True, prec=dfft.FLOAT)) == 0
    monkeypatch.setenv("DFFT_VARIANT", "5")                                                      # an alternate tuning of 512: no
    assert _code(mk(n0=512)) == -3                                                               # convolution kinds
    monkeypatch.delenv("DFFT_VARIANT")
    assert _code(mk(n0=512)) == 0
    # execute-time rejections
    p = dfft.fft_mpi_plan_dft_convolve_3d(16, 16, 16, i, o, None, 0, 1, dfft.DOUBLE, dfft.DRY_RUN)
    assert _code(p.execute) == -1
    assert _code(lambda: p.execute_stage(0)) == -1
    assert _code(lambda: p.execute_host(i, o)) == -1
    assert _code(lambda: p.execute_convolve(None)) == -1
    assert _code(lambda: p.execute_convolve(fake(0, MULT) + 8)) == -1
    assert _code(lambda: p.execute_convolve(fake(0, MULT) + 16)) == 0
    p.destroy()
    p = dfft.fft_mpi_plan_dft_convolve_3d(16, 16, 16, i, o, None, 0, 1, dfft.FLOAT, dfft.DRY_RUN, real=True)
    assert _code(lambda: p.execute_convolve(fake(0, MULT) + 4)) == -1
    assert _code(lambda: p.execute_convolve(fake(0, MULT) + 8)) == 0
    p.destroy()
    for real in (False, True):
        q = (dfft.fft_mpi_plan_dft_r2c_3d if real else dfft.fft_mpi_plan_dft_c2c_3d)(16, 16, 16, i, o, None, 0, 1, dfft.FORWARD, dfft.DOUBLE, dfft.DRY_RUN)
        assert _code(lambda: q.execute_convolve(fake(0, MULT))) == -1
        q.destroy()


# ---- the bound of the GPU tests ------------------------------------------------------------------------------------------
CONV_L2_K, CONV_LINF_K = 2 * ldfft.REL_L2_K, 2 * ldfft.LINF_K


def ld_convolve(A, M, fwd_dtype=np.clongdouble, perturb=None):
    S = ldfft.fftn(A, dtype=fwd_dtype, perturb=perturb).astype(np.clongdouble) * np.asarray(M).astype(np.clongdouble)
    return ldfft.fftn(S, sign=1)


@pytest.mark.parametrize("shape", [(16, 32, 64), (8, 12, 256)])
def test_bound_accepts_numpy_and_rejects_a_40_bit_twiddle_stage(shape):
    rng = np.random.default_rng(11)
    A = rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    M = rng.uniform(0.5, 2.0, shape) * np.exp(2j * np.pi * rng.uniform(size=shape))
    ref = ld_convolve(A, M)
    ntot, eps = A.size, ldfft.EPS["double"]
    r = ldfft.ratios(np.fft.ifftn(np.fft.fftn(A) * M) * ntot, ref, eps, ntot)
    assert r[0] <= CONV_L2_K and r[1] <= CONV_LINF_K, r
    bad = ld_convolve(A, M, np.complex128, perturb=(1, 40))
    r_bad = ldfft.ratios(bad, ref, eps, ntot)
    assert r_bad[0] > CONV_L2_K and r_bad[1] > CONV_LINF_K, r_bad
