"""R2C / C2R slab transforms (dfft_plan_r2c_3d) on the GPU.

The real Z pass (fft_real.cuh) transforms two real lines as one complex line and separates the two half spectra, so every
tuned z length is run through P = 1 plans with short y and x axes, odd and even local line counts, in both precisions,
against a long-double reference (tests/ldfft.py) with the bounds of test_gpu_tma_matrix.py: rel_l2 <= 1.0 * eps * log2(Ntot)
and max error / rms(ref) <= 4 * eps * log2(Ntot).  The backward input is NOT Hermitian: the C2R result must be what
numpy.fft.irfftn(., s) * Ntot returns, i.e. the imaginary parts at z = 0 and z = n2/2 are ignored.  Each case prints
"R2C-RATIO" lines.

Outputs are NaN-prefilled and fenced with canaries exactly at the complex / real count; plans execute three times.  Then
full cubes (512^3 fp64, 768^3 fp32, 100x96x1000 fp64) against scipy's multi-threaded fp64 FFT, the round trip, the natural
spectrum, the host entry points, default against DFFT_NO_TMA, and P = 2, 4, 8 device-threads (skipped on a smaller box)."""
import faulthandler
import sys
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from ld_harness import ratios64  # noqa: E402

FWD, BWD = dfft.FORWARD, dfft.BACKWARD
RDT = {dfft.DOUBLE: (np.float64, torch.float64), dfft.FLOAT: (np.float32, torch.float32)}
CDT = {dfft.DOUBLE: (np.complex128, torch.complex128), dfft.FLOAT: (np.complex64, torch.complex64)}
EPS = {dfft.DOUBLE: ldfft.EPS["double"], dfft.FLOAT: ldfft.EPS["float"]}
CANARY = 64
WORST = {}


@pytest.fixture(autouse=True)
def _watchdog():
    faulthandler.dump_traceback_later(600, exit=True, file=sys.stderr)
    yield
    faulthandler.cancel_dump_traceback_later()


def need(P):
    if torch.cuda.device_count() < P:
        pytest.skip(f"needs {P} GPUs, box has {torch.cuda.device_count()}")


def fenced(host, tdt, dev=0):
    """device arena [canary | data | canary] holding `host` (flat numpy, or an int length for a NaN-filled output)"""
    d = torch.device("cuda", dev)
    n = host if isinstance(host, int) else host.size
    rng = np.random.default_rng(99)
    pat = rng.standard_normal(2 * CANARY) if not tdt.is_complex else rng.standard_normal(2 * CANARY) + 1j * rng.standard_normal(2 * CANARY)
    pat = torch.from_numpy(pat).to(tdt).to(d)
    arena = torch.empty(2 * CANARY + n, dtype=tdt, device=d)
    arena[:CANARY], arena[CANARY + n:] = pat[:CANARY], pat[CANARY:]
    if isinstance(host, int):
        arena[CANARY: CANARY + n] = float("nan")
    else:
        arena[CANARY: CANARY + n] = torch.from_numpy(host).to(d)
    return arena, arena[:CANARY].clone(), arena[CANARY + n:].clone()


def run_plan(n0, n1, n2, prec, direction, dev_in, flags=0, repeat=3, info=None):
    """one P = 1 plan on fenced buffers, executed `repeat` times; returns the output as numpy (info: dict that receives the
    plan's tma_mask)"""
    torch.cuda.set_device(0)
    rc, cc = dfft.local_size_r2c_3d(n0, n1, n2, 1, 0)
    in_t, out_t = (RDT[prec][1], CDT[prec][1]) if direction == FWD else (CDT[prec][1], RDT[prec][1])
    n_in, n_out = (rc, cc) if direction == FWD else (cc, rc)
    assert dev_in.size == n_in
    a_in, _, _ = fenced(dev_in, in_t)
    a_out, lo, hi = fenced(n_out, out_t)
    inp, out = a_in[CANARY: CANARY + n_in], a_out[CANARY: CANARY + n_out]
    plan = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, inp.data_ptr(), out.data_ptr(), None, 0, 1, direction, prec, flags)
    assert (plan.in_count, plan.out_count) == (n_in, n_out)
    first = None
    for _ in range(repeat):
        plan.execute()
        plan.synchronize()
        cur = out.cpu().numpy().copy()
        if first is None:
            first = cur
        else:
            assert np.array_equal(cur.view(np.uint8), first.view(np.uint8)), "executes differ"
    t = plan.timings()
    assert len(t) == 5 and plan.pass_timings()[0] > 0
    if info is not None:
        info["tma_mask"] = plan.tma_mask
    plan.destroy()
    torch.cuda.synchronize()
    assert torch.equal(a_out[:CANARY], lo) and torch.equal(a_out[CANARY + n_out:], hi), "canary overwritten"
    assert torch.equal(inp.cpu(), torch.from_numpy(dev_in)), "input changed"
    assert not np.isnan(first).any(), "unwritten output"
    return first


def ld_r2c(x):
    """long-double rfftn: [x][y][z] real -> [x][y][nzh]"""
    y = ldfft.fftn(x.astype(np.longdouble) + 0j)
    return y[:, :, : x.shape[2] // 2 + 1]


def ld_c2r(S, n2):
    """long-double irfftn(S, s=(.., .., n2)) * Ntot: inverse x, y, then the Hermitian extension along z (imaginary parts of
    z = 0 and z = n2/2 dropped), inverse z, real part"""
    y = ldfft.fft(ldfft.fft(S.astype(np.clongdouble), 0, +1), 1, +1)
    H = n2 // 2 + 1
    y[:, :, 0] = y[:, :, 0].real
    if n2 % 2 == 0:
        y[:, :, H - 1] = y[:, :, H - 1].real
    full = np.empty(S.shape[:2] + (n2,), dtype=np.clongdouble)
    full[:, :, :H] = y
    full[:, :, H:] = np.conj(y[:, :, 1: n2 - H + 1][:, :, ::-1])
    return ldfft.fft(full, 2, +1).real


def check(got, ref, prec, ntot, what):
    big = np.asarray(ref).dtype in (np.float64, np.complex128)
    rl2, linf = (ratios64 if big else ldfft.ratios)(got, ref, EPS[prec], ntot)
    print(f"R2C-RATIO {what} rel_l2 {rl2:.3f} linf {linf:.3f}")
    key = (what.split()[0], prec)
    WORST[key] = max(WORST.get(key, (0, 0)), (rl2, linf))
    assert rl2 <= ldfft.REL_L2_K and linf <= ldfft.LINF_K, (what, rl2, linf)


def tuned(prec):
    return [n for n in dfft.supported_lengths(prec) if dfft.length_kind(n, prec) == 2]


@pytest.mark.parametrize("prec", [dfft.DOUBLE, dfft.FLOAT])
def test_every_tuned_z_length(prec):
    rdt, cdt = RDT[prec][0], CDT[prec][0]
    for n2 in tuned(prec):
        for n0, n1 in ((3, 5), (2, 4)):      # 15 lines: the last pair has no partner line; 8 lines: every pair complete
            rng = np.random.default_rng(n2 * 10 + n0)
            ntot = n0 * n1 * n2
            x = rng.standard_normal((n0, n1, n2)).astype(rdt)
            want = ld_r2c(x).transpose(1, 2, 0).reshape(-1)
            got = run_plan(n0, n1, n2, prec, FWD, x.reshape(-1))
            check(got, want, prec, ntot, f"fwd n2={n2} {n0}x{n1} prec={prec}")
            H = n2 // 2 + 1
            S = (rng.standard_normal((n0, n1, H)) + 1j * rng.standard_normal((n0, n1, H))).astype(cdt)   # not Hermitian
            want = ld_c2r(S, n2).reshape(-1)
            got = run_plan(n0, n1, n2, prec, BWD, np.ascontiguousarray(S.transpose(1, 2, 0)).reshape(-1), dfft.SCALE_BACKWARD if n0 == 2 else 0)
            if n0 == 2:
                want = want / np.longdouble(ntot)
            check(got, want, prec, ntot, f"bwd n2={n2} {n0}x{n1} prec={prec}")


def sp_rfftn(A):
    import scipy.fft
    return scipy.fft.rfftn(A.astype(np.float64), workers=-1)


@pytest.mark.parametrize("n0,n1,n2,prec", [(512, 512, 512, dfft.DOUBLE), (768, 768, 768, dfft.FLOAT), (100, 96, 1000, dfft.DOUBLE)])
def test_full_cubes(n0, n1, n2, prec):
    import scipy.fft
    rdt, cdt = RDT[prec][0], CDT[prec][0]
    ntot = n0 * n1 * n2
    rng = np.random.default_rng(n0 + n2)
    A = rng.standard_normal((n0, n1, n2)).astype(rdt)
    ref = sp_rfftn(A)
    spec = run_plan(n0, n1, n2, prec, FWD, A.reshape(-1))
    check(spec, ref.transpose(1, 2, 0).reshape(-1), prec, ntot, f"cube-fwd {n0}x{n1}x{n2} prec={prec}")
    del ref
    # round trip with SCALE_BACKWARD
    back = run_plan(n0, n1, n2, prec, BWD, spec, dfft.SCALE_BACKWARD, repeat=1)
    check(back, A.reshape(-1).astype(np.float64), prec, ntot, f"cube-roundtrip {n0}x{n1}x{n2} prec={prec}")
    del back
    # C2R of a non-Hermitian spectrum equals irfftn * Ntot
    H = n2 // 2 + 1
    S = (rng.standard_normal((n0, n1, H)) + 1j * rng.standard_normal((n0, n1, H))).astype(cdt)
    got = run_plan(n0, n1, n2, prec, BWD, np.ascontiguousarray(S.transpose(1, 2, 0)).reshape(-1), repeat=1)
    want = scipy.fft.irfftn(S.astype(np.complex128), s=(n0, n1, n2), workers=-1) * ntot
    check(got, want.reshape(-1), prec, ntot, f"cube-c2r {n0}x{n1}x{n2} prec={prec}")
    del want, got
    # natural spectrum, both directions
    nat = run_plan(n0, n1, n2, prec, FWD, A.reshape(-1), dfft.NATURAL_SPECTRUM, repeat=1)
    assert np.array_equal(nat.reshape(n0, n1, H), spec.reshape(n1, H, n0).transpose(2, 0, 1)), "natural spectrum differs"
    back = run_plan(n0, n1, n2, prec, BWD, nat, dfft.NATURAL_SPECTRUM | dfft.SCALE_BACKWARD, repeat=1)
    check(back, A.reshape(-1).astype(np.float64), prec, ntot, f"cube-natural-roundtrip {n0}x{n1}x{n2} prec={prec}")


def test_host_entry_points_with_pinned_buffers():
    n0, n1, n2 = 64, 48, 100
    rc, cc = dfft.local_size_r2c_3d(n0, n1, n2, 1, 0)
    rng = np.random.default_rng(3)
    A = rng.standard_normal(rc)
    h_in = torch.from_numpy(A).pin_memory()
    h_spec = torch.full((cc,), float("nan"), dtype=torch.complex128).pin_memory()
    h_back = torch.full((rc,), float("nan"), dtype=torch.float64).pin_memory()
    d_in = torch.zeros(rc, dtype=torch.float64, device="cuda")
    d_out = torch.zeros(cc, dtype=torch.complex128, device="cuda")
    fwd = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, d_in.data_ptr(), d_out.data_ptr(), None, 0, 1, FWD)
    bwd = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, d_out.data_ptr(), d_in.data_ptr(), None, 0, 1, BWD, dfft.DOUBLE, dfft.SCALE_BACKWARD)
    fwd.execute_host(h_in.data_ptr(), h_spec.data_ptr())
    ref = np.fft.rfftn(A.reshape(n0, n1, n2)).transpose(1, 2, 0).reshape(-1)
    assert np.abs(h_spec.numpy() - ref).max() <= 1e-12 * np.abs(ref).max()
    bwd.execute_host_async(h_spec.data_ptr(), h_back.data_ptr())
    bwd.synchronize()
    assert np.abs(h_back.numpy() - A).max() <= 1e-13
    fwd.destroy()
    bwd.destroy()


def test_512_default_matches_no_tma_bit_for_bit():
    """A guard for when a TMA pass becomes reachable for R2C plans.  Today none is: the Z pass is always the real-data kernel,
    and the Y and X passes need nzh = n2/2 + 1 to be a multiple of the TMA entry's tile width, which 257 is not (for every even
    tuned n2, nzh is odd).  So both plans must report tma_mask 0 and launch the same kernels; once a TMA pass is used for R2C
    the masks differ and the bit-for-bit comparison becomes the real check (C2C is bit-identical at 512 the same way)."""
    n = 512
    A = np.random.default_rng(5).standard_normal(n ** 3)
    ia, ib = {}, {}
    a = run_plan(n, n, n, dfft.DOUBLE, FWD, A, repeat=1, info=ia)
    b = run_plan(n, n, n, dfft.DOUBLE, FWD, A, dfft.NO_TMA, repeat=1, info=ib)
    assert (ia["tma_mask"], ib["tma_mask"]) == (0, 0)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


# short z lengths with far more tiles than resident CTAs (132 SMs x at most 16 CTAs of these sizes): every CTA runs several
# tiles, so the end-of-tile barrier and the exchange-buffer reuse across tiles of the grid-stride loop are exercised (the
# per-length test above has fewer tiles than CTAs).  n0 x n1 = 525525 (z <= 16) or 275275 lines, both odd
@pytest.mark.parametrize("prec", [dfft.DOUBLE, dfft.FLOAT])
@pytest.mark.parametrize("n2", [4, 9, 10, 16, 24, 64, 125, 243])
def test_grid_stride_many_tiles(prec, n2):
    import scipy.fft
    n0, n1 = (1001, 525) if n2 <= 16 else (1001, 275)
    rdt, cdt = RDT[prec][0], CDT[prec][0]
    ntot = n0 * n1 * n2
    rng = np.random.default_rng(n2)
    A = rng.standard_normal((n0, n1, n2)).astype(rdt)
    got = run_plan(n0, n1, n2, prec, FWD, A.reshape(-1), repeat=2)
    check(got, sp_rfftn(A).transpose(1, 2, 0).reshape(-1), prec, ntot, f"many-tiles-fwd n2={n2} prec={prec}")
    H = n2 // 2 + 1
    S = (rng.standard_normal((n0, n1, H)) + 1j * rng.standard_normal((n0, n1, H))).astype(cdt)
    got = run_plan(n0, n1, n2, prec, BWD, np.ascontiguousarray(S.transpose(1, 2, 0)).reshape(-1), repeat=2)
    want = scipy.fft.irfftn(S.astype(np.complex128), s=(n0, n1, n2), workers=-1) * ntot
    check(got, want.reshape(-1), prec, ntot, f"many-tiles-bwd n2={n2} prec={prec}")


def run_multi(n0, n1, n2, P, direction, inputs, flags):
    """P device-threads of one process; inputs[d] = device d's input slab; returns each device's output as numpy"""
    comm = dfft.LocalComm(P)
    res, errs = [None] * P, []
    barrier = threading.Barrier(P)

    def worker(d):
        try:
            torch.cuda.set_device(d)
            rc, cc = dfft.local_size_r2c_3d(n0, n1, n2, P, d)
            n_out = cc if direction == FWD else rc
            inp = torch.from_numpy(inputs[d]).to(f"cuda:{d}")
            out = torch.full((n_out,), float("nan"), dtype=torch.complex128 if direction == FWD else torch.float64, device=f"cuda:{d}")
            plan = dfft.fft_mpi_plan_dft_r2c_3d(n0, n1, n2, inp.data_ptr(), out.data_ptr(), comm, d, P, direction, dfft.DOUBLE, flags)
            assert plan.exchange == flags & 3
            for _ in range(2):
                plan.execute()
            plan.synchronize()
            res[d] = out.cpu().numpy()
            barrier.wait()
            plan.destroy()
        except Exception:
            import traceback
            errs.append(traceback.format_exc())
            barrier.abort()

    th = [threading.Thread(target=worker, args=(d,)) for d in range(P)]
    [t.start() for t in th]
    [t.join() for t in th]
    comm.destroy()
    assert not errs, "\n".join(errs)
    return res


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("P,n0,n1,n2", [(2, 64, 64, 64), (2, 30, 21, 9), (4, 128, 128, 128), (4, 12, 10, 100), (8, 64, 64, 64), (8, 30, 22, 243)])
def test_multi_gpu_vs_numpy(mode, P, n0, n1, n2):
    need(P)
    flags = dfft.EXCHANGE_P2P if mode == "p2p" else dfft.EXCHANGE_NCCL
    rng = np.random.default_rng(P * 7 + n2)
    A = rng.standard_normal((n0, n1, n2))
    xd, yd, H = -(-n0 // P), -(-n1 // P), n2 // 2 + 1
    ref = np.fft.rfftn(A)
    got = run_multi(n0, n1, n2, P, FWD, [np.ascontiguousarray(A[d * xd:(d + 1) * xd]).reshape(-1) for d in range(P)], flags)
    for d in range(P):
        want = ref[:, d * yd:(d + 1) * yd, :].transpose(1, 2, 0).reshape(-1)
        assert np.abs(got[d] - want).max() <= 1e-12 * np.log2(A.size) * np.abs(ref).max(), (d, mode)
    S = rng.standard_normal((n0, n1, H)) + 1j * rng.standard_normal((n0, n1, H))
    bref = np.fft.irfftn(S, s=(n0, n1, n2), axes=(0, 1, 2)) * A.size
    got = run_multi(n0, n1, n2, P, BWD, [np.ascontiguousarray(S[:, d * yd:(d + 1) * yd, :].transpose(1, 2, 0)).reshape(-1) for d in range(P)], flags)
    for d in range(P):
        want = bref[d * xd:(d + 1) * xd].reshape(-1)
        assert np.abs(got[d] - want).max() <= 1e-12 * np.log2(A.size) * np.abs(bref).max(), (d, mode)


def test_zz_report_worst_ratios():
    for (what, prec), (rl2, linf) in sorted(WORST.items()):
        print(f"R2C-WORST {what} prec={prec} rel_l2 {rl2:.3f} linf {linf:.3f}")
