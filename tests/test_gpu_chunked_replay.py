"""The multi-device pass kinds on one H100: the chunked and peer-store kernels against the long-double reference.

The kernels of Y_CO, Y_CI, XB_CO, XCONV_CO and of the fused t0 with the chunked store / load (FK_ZY_CO, FK_YZ_CI) only run
when a plan spans several devices.  tests/gpu_replay.py replays the records of the P per-device DFFT_DRY_RUN plans on GPU 0,
one launch per record (per fused pair) in dependency order, every virtual device's buffers in their own fenced, NaN-prefilled
allocations.  Each case checks
  (a) the gathered output slabs against ldfft.fftn of the precision-rounded input (rel_l2 <= 1, linf <= 4 in units of
      eps * log2(Ntot)); convolve plans against the long-double convolution at twice those bounds; cases too large for the
      long-double reference against scipy's fp64 transform (ld_harness.ratios64);
  (b) bitwise equality with the one-device plan of the same shape and flags (NO_TMA; fused t0 where the replayed schedule
      fuses it, NO_FUSE otherwise): every line runs the same radix schedule whatever the tiling (s_rad for the local and the
      peer-store Y configurations, x_rad for both X kinds), and the fused and two-sweep t0 are bit-identical (DESIGN.md 4);
  (c) no NaN left in an output slab, every canary intact, bufferDev1 and the multiplier bitwise unchanged (gpu_replay).
The in-kernel synchronisation of fused_yx / fused3 and the P2P arrival flags are not exercised: nothing here runs two
devices' kernels at once.  The worst ratios per record kind and precision are printed as "REPLAY-WORST" lines."""
import faulthandler
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from gpu_replay import MULT, Replay, slab_outputs  # noqa: E402
from ld_harness import CDT, EPS, bits, layouts, ratios64, run_fenced  # noqa: E402
from oracle import SlabGeometry  # noqa: E402
from test_dry_run import BUF1, IN, dry_ops, fake  # noqa: E402

DOUBLE, FLOAT, FWD, BWD = dfft.DOUBLE, dfft.FLOAT, dfft.FORWARD, dfft.BACKWARD
P2P, NCCL, NO_FUSE, NO_TMA = dfft.EXCHANGE_P2P, dfft.EXCHANGE_NCCL, dfft.NO_FUSE, dfft.NO_TMA
PN = {DOUBLE: "fp64", FLOAT: "fp32"}
LD_MAX = 1 << 21          # elements up to which the long-double reference is used
MODES = {"p2p": P2P, "p2p-nofuse": P2P | NO_FUSE, "nccl": NCCL}
# generic (run-time scheduled) lengths: their chunked kinds are kernels of their own (fft_generic_kernel with the chunk tables)
GENERIC = [7, 14, 22, 1001]
WORST = {}
SEEN = {}
_ONE = {}


@pytest.fixture(autouse=True)
def _watchdog():
    faulthandler.dump_traceback_later(900, exit=True, file=sys.stderr)
    yield
    faulthandler.cancel_dump_traceback_later()


def tuned(prec):
    return [n for n in dfft.supported_lengths(prec) if dfft.length_kind(n, prec) == 2]


def kinds(ops):
    """the record kinds of a replay, a fused pair named by the kernel it runs as"""
    out = set()
    for o in ops:
        for k, op in enumerate(o):
            if op["op"] == "fusedZ" and k + 1 < len(o) and o[k + 1]["op"] == "fusedY":
                out.add("FK_ZY_CO" if "co" in o[k + 1] else "FK_ZY")
            elif op["op"] == "fusedY" and k + 1 < len(o) and o[k + 1]["op"] == "fusedZ":
                out.add("FK_YZ_CI" if "ci" in op else "FK_YZ")
            elif op["op"] not in ("alltoall", "fusedZ", "fusedY"):
                out.add(op["op"])
    return out


def note(ops, prec, r, label, family="c2c"):
    """print a case's ratios and fold them into the worst per (family, kind, precision); returns the case's kinds.  The
    convolve cases are their own family: they are held to twice the bounds"""
    print("REPLAY-RATIO %-60s rel_l2 %6.3f  linf %6.3f" % (label, r[0], r[1]))
    ks = kinds(ops)
    for k in ks:
        w = WORST.get((family, k, prec), (0.0, 0.0))
        WORST[family, k, prec] = (max(w[0], r[0]), max(w[1], r[1]))
        SEEN[family, k, prec] = SEEN.get((family, k, prec), 0) + 1
    return ks


def split_input(dev_in, g, direction):
    """the P bufferDev1 slabs of the one-device layout: x-slabs [x_l][y][z] forward, y-slabs [y_l][z][x] backward"""
    if direction == FWD:
        rows = dev_in.reshape(g.n0, -1)
        return [rows[d * g.xd: d * g.xd + g.n0l(d)].reshape(-1) for d in range(g.P)]
    rows = dev_in.reshape(g.n1, -1)
    return [rows[d * g.yd: d * g.yd + g.n1l(d)].reshape(-1) for d in range(g.P)]


def one_device(shape, prec, direction, dev_in, fused, scale, inplace):
    """output of the P = 1 plan with the replayed schedule's t0 (cached: it does not depend on P or the exchange)"""
    key = (shape, prec, direction, fused, scale, inplace, dev_in.tobytes()[:64])
    if key not in _ONE:
        flags = NO_TMA | (dfft.FORCE_FUSE if fused else NO_FUSE) | (dfft.SCALE_BACKWARD if scale else 0)
        while len(_ONE) >= 4 or (_ONE and dev_in.size > LD_MAX):
            _ONE.pop(next(iter(_ONE)))
        _ONE[key] = run_fenced(shape, prec, direction, dev_in, flags, inplace=inplace, repeat=1)[0]
    return _ONE[key]


def replay_c2c(shape, P, prec, direction, flags, scale=False, inplace=False, seed=None, label="", min_tiles=0, tiles_of=()):
    """one replayed C2C case: checks (a), (b), (c); returns the records (None: the geometry leaves a device empty).  min_tiles:
    every record of a kind in `tiles_of` has at least that many tiles"""
    n0, n1, n2 = shape
    g = SlabGeometry(n0, n1, n2, P)
    if g.last_n0 < 1 or g.last_n1 < 1:
        return None
    seed = seed if seed is not None else n0 * 7 + n1 * 13 + n2
    flags |= NO_TMA | (dfft.SCALE_BACKWARD if scale else 0)
    ops, fused = dry_ops(n0, n1, n2, P, direction, flags, prec, inplace)
    assert len(set(fused)) == 1
    ntot = n0 * n1 * n2
    big = ntot > LD_MAX
    if big:
        rng = np.random.default_rng(seed)
        x = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(CDT[prec][0])
        dev_in = x.reshape(-1) if direction == FWD else np.ascontiguousarray(x.transpose(1, 2, 0)).reshape(-1)
        want = None
    else:
        dev_in, want = layouts(shape, seed, prec, direction, scale=scale)
    slabs = split_input(dev_in, g, direction)
    init = {(d, BUF1): slabs[d] for d in range(P)}
    if inplace:
        init.update({(d, IN): slabs[d] for d in range(P)})
    if min_tiles:
        sub = [op["ntiles"] for o in ops for op in o if op["op"] in tiles_of]
        assert sub and min(sub) >= min_tiles, (label, sub, min_tiles)
    rep = Replay(g, ops, prec, init)
    launches = rep.run()
    assert launches == sum(1 for o in ops for op in o if op["op"] not in ("alltoall", "fusedY", "fusedZ")) + \
        sum(1 for o in ops for op in o if op["op"] == "fusedZ")
    got = rep.contents(slab_outputs(g, direction, inplace))
    out = np.concatenate([got[k] for k in sorted(got)])
    del rep
    torch.cuda.empty_cache()
    # (b) the one-device plan, bit for bit
    ref1 = one_device(shape, prec, direction, dev_in, fused[0], scale, inplace)
    assert np.array_equal(bits(out), bits(ref1)), ("not bit-identical to the one-device plan", label)
    # (a) the reference
    if big:
        import scipy.fft as sf
        x64 = x.astype(np.complex128)
        y = sf.fftn(x64) if direction == FWD else sf.ifftn(x64) * ntot
        if scale:
            y = y / ntot
        ref = np.ascontiguousarray(y.transpose(1, 2, 0)) if direction == FWD else y
        r = ratios64(out, ref, EPS[prec], ntot)
    else:
        r = ldfft.ratios(out, want, EPS[prec], ntot)
    note(ops, prec, r, label)
    assert r[0] <= ldfft.REL_L2_K and r[1] <= ldfft.LINF_K, (label, r)
    return ops


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
def test_every_length_as_the_exchanged_y_axis(prec):
    """9 x N x 10 slabs: the Y pass with the packed / peer store (Y_CO, ragged p_C tiles where p_C does not divide 10) and the
    inverse Y pass with the chunked load (Y_CI), over 2 and 3 devices (uneven yd), P2P and NCCL, both directions; the backward
    cases alternate scaled / in place"""
    seen = set()
    lengths = tuned(prec)
    for i, n in enumerate(lengths + GENERIC):
        for P in (2, 3):
            for mode in ("p2p", "nccl"):
                for direction in (FWD, BWD):
                    scale = direction == BWD and i % 2 == 0
                    inplace = (i + P) % 3 == 0
                    ops = replay_c2c((9, n, 10), P, prec, direction, MODES[mode], scale, inplace,
                                     label=f"n1={n} 9x{n}x10 P={P} {mode} {'fwd' if direction == FWD else 'bwd'}{' scaled' if scale else ''}{' inplace' if inplace else ''}")
                    if ops is not None:
                        seen |= {(k, op["N"]) for o in ops for op in o for k in [op["op"]] if "ci" in op or "co" in op}
    for k in {"Y_CO", "Y_CI"} - {"XF"}:
        assert {n for kk, n in seen if kk == k} >= set(lengths + GENERIC) - {2}, (k, sorted(n for kk, n in seen if kk == k))


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
def test_every_length_as_the_exchanged_x_axis(prec):
    """N x 9 x 10 slabs: the forward X pass (XF) over the received planes and the backward X pass with the peer store
    (XB_CO), over 2 and 3 devices (uneven xd), P2P and NCCL, both directions"""
    seen = set()
    lengths = tuned(prec)
    for i, n in enumerate(lengths + GENERIC):
        for P in (2, 3):
            for mode in ("p2p", "nccl"):
                for direction in (FWD, BWD):
                    scale = direction == BWD and i % 2 == 1
                    inplace = (i + P) % 3 == 1
                    ops = replay_c2c((n, 9, 10), P, prec, direction, MODES[mode], scale, inplace,
                                     label=f"n0={n} {n}x9x10 P={P} {mode} {'fwd' if direction == FWD else 'bwd'}{' scaled' if scale else ''}{' inplace' if inplace else ''}")
                    if ops is not None:
                        seen |= {(k, op["N"]) for o in ops for op in o for k in [op["op"]] if "ci" in op or "co" in op}
    for k in {"XF", "XB_CO"} - {"XF"}:
        assert {n for kk, n in seen if kk == k} >= set(lengths + GENERIC) - {2}, (k, sorted(n for kk, n in seen if kk == k))


def fused_lengths(prec, P):
    out = []
    for n in tuned(prec):
        ops, fused = dry_ops(P, n, n, P, FWD, P2P | NO_TMA, prec)
        if fused[0]:
            out.append(n)
    return out


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
def test_fused_t0_with_the_chunked_store_and_load(prec):
    """square planes n0 x N x N, n0 = P or P + 1: FK_ZY_CO forward and FK_YZ_CI backward for every length with a fused entry,
    and the same plans with NO_FUSE (Z + Y_CO, Y_CI + Z); over 2 GB of buffers the reference is scipy's fp64 transform"""
    lengths = fused_lengths(prec, 2)
    assert lengths, "no fused entry"
    for i, n in enumerate(lengths):
        P = 3 if i % 2 and SlabGeometry(3, n, n, 3).last_n1 >= 1 else 2   # (4 rows over 3 devices would leave the last one empty)
        n0 = P + 1 if P == 2 and (i // 2) % 2 else P          # (3 planes over 3 devices would leave the last one empty)
        esz = 16 if prec == DOUBLE else 8
        if 3 * n0 * n * n * esz > 2 << 30:
            n0 = P
        for mode in ("p2p", "p2p-nofuse"):
            for direction in (FWD, BWD):
                scale = direction == BWD and mode == "p2p"
                ops = replay_c2c((n0, n, n), P, prec, direction, MODES[mode], scale,
                                 label=f"{n0}x{n}x{n} P={P} {mode} {'fwd' if direction == FWD else 'bwd'}{' scaled' if scale else ''}")
                assert ops is not None
                if mode == "p2p":
                    assert ("FK_ZY_CO" if direction == FWD else "FK_YZ_CI") in kinds(ops), (n, kinds(ops))


PIPE_CASES = [("p2p", 2, (8, 128, 128), None, None), ("p2p", 3, (10, 9, 128), None, None), ("p2p", 2, (64, 64, 64), "2", None),
              ("p2p", 2, (64, 64, 64), "2", "streams"), ("p2p", 3, (6, 64, 64), "4", "streams"), ("nccl", 2, (8, 16, 128), None, None),
              ("nccl", 2, (8, 8, 64), "2", None), ("p2p", 3, (9, 256, 256), "4", "streams")]


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
@pytest.mark.parametrize("mode,P,shape,parts,pipe_mode", PIPE_CASES)
def test_stream_pipelined_schedules(monkeypatch, prec, mode, P, shape, parts, pipe_mode):
    """FORCE_PIPELINE: z-parts of the Y pass with part-major peer stores / packed send parts, per-part all-to-alls, X parts;
    backward: XB_CO parts, Y_CI parts, the last one fused with the inverse Z pass.  DFFT_PIPE_MODE=streams keeps the cube
    off the fused Y + X kernel (whose records replay as Y_CO + XF anyway)"""
    for var, val in (("DFFT_PARTS", parts), ("DFFT_PIPE_MODE", pipe_mode)):
        if val:
            monkeypatch.setenv(var, val)
        else:
            monkeypatch.delenv(var, raising=False)
    for direction in (FWD, BWD):
        ops = replay_c2c(shape, P, prec, direction, MODES[mode] | dfft.FORCE_PIPELINE, scale=direction == BWD,
                         label=f"pipelined {mode} P={P} {'x'.join(map(str, shape))} parts={parts} {pipe_mode} {'fwd' if direction == FWD else 'bwd'}")
        names = [op["op"] for op in ops[0]]
        assert names.count("XF" if direction == FWD else "XB_CO") >= 2, names


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
def test_many_tiles_per_resident_cta(prec):
    """long z rows: the Y pass of length 16 (200 x 16 x 4096) and the X pass of length 8 (8 x 256 x 4096) have at least 3 tiles
    for every CTA an H100 can hold resident (132 SMs x 32), so every CTA of those launches loops over several tiles"""
    need = 3 * 132 * 32
    for shape, subject in (((200, 16, 4096), ("Y_CO", "Y_CI")), ((8, 256, 4096), ("XF", "XB", "XB_CO"))):
        for mode in ("p2p", "nccl"):
            for direction in (FWD, BWD):
                replay_c2c(shape, 2, prec, direction, MODES[mode], min_tiles=need, tiles_of=subject,
                           label=f"many tiles {'x'.join(map(str, shape))} P=2 {mode} {'fwd' if direction == FWD else 'bwd'}")


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
@pytest.mark.parametrize("P,shape,mode", [(2, (16, 12, 10), "p2p"), (3, (12, 10, 9), "p2p"), (2, (16, 16, 16), "p2p"),
                                          (3, (24, 32, 32), "p2p"), (3, (12, 10, 9), "nccl"), (2, (64, 64, 64), "p2p-nofuse")])
def test_convolve_c2c(prec, P, shape, mode):
    """the fused X pass with the peer store (XCONV_CO) between the forward and backward halves, random multiplier; against the
    long-double convolution and, bit for bit, the one-device convolve plan"""
    from test_gpu_convolve import K_L2, K_LINF, ld_conv, multipliers, run_conv
    n0, n1, n2 = shape
    g = SlabGeometry(n0, n1, n2, P)
    flags = MODES[mode] | NO_TMA
    rng = np.random.default_rng(P * 1000 + n0)
    A = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(CDT[prec][0])
    M = multipliers(n0, n1, n2, prec, n0 + P)["rand"]
    plans = [dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, fake(d, IN), fake(d, 2), None, d, P, prec, flags | dfft.DRY_RUN) for d in range(P)]
    ops = []
    for d, p in enumerate(plans):
        p.execute_convolve(fake(d, MULT))
        ops.append(p.recorded_ops())
    fwd_fused = any(op["op"] == "fusedZ" and op["phase"] == 0 for op in ops[0])
    for p in plans:
        p.destroy()
    init = {}
    for d in range(P):
        init[d, BUF1] = A[d * g.xd: d * g.xd + g.n0l(d)].reshape(-1)
        init[d, MULT] = np.ascontiguousarray(M[:, d * g.yd: d * g.yd + g.n1l(d), :]).reshape(-1)
    rep = Replay(g, ops, prec, init, nphases=4)
    rep.run()
    got = rep.contents({(d, 2): g.n0l(d) * n1 * n2 for d in range(P)})
    out = np.concatenate([got[d, 2] for d in range(P)]).reshape(shape)
    del rep
    ref1 = run_conv(A, {"rand": M}, prec, False, NO_TMA | (dfft.FORCE_FUSE if fwd_fused else NO_FUSE))["rand"]
    assert np.array_equal(bits(out), bits(ref1)), "not bit-identical to the one-device convolve plan"
    r = ldfft.ratios(out, ld_conv(A, M, False), EPS[prec], A.size)
    ks = note(ops, prec, r, f"convolve {'x'.join(map(str, shape))} P={P} {mode}", family="convolve")
    assert ("XCONV" if mode == "nccl" else "XCONV_CO") in ks, ks
    assert r[0] <= K_L2 and r[1] <= K_LINF, r


def test_zz_report_worst_ratios():
    """the table of the cases run before it in this process (each test asserts the kinds it is about itself)"""
    if not WORST:
        pytest.skip("no replay case ran in this process")
    for (fam, k, prec), (rl2, linf) in sorted(WORST.items()):
        print("REPLAY-WORST %-8s %-9s %s rel_l2 %.3f linf %.3f  (%d cases)" % (fam, k, PN[prec], rl2, linf, SEEN[fam, k, prec]))
