"""Spectral convolution plans (dfft_plan_convolve_c2c_3d / dfft_plan_convolve_r2c_3d) on the GPU.

The fused X pass (fft_conv_kernel: forward FFT along x, multiply, inverse FFT along x in one column pass) is run for every tuned x
length on thin slabs, both precisions, both variants, default and NO_TMA | NO_FUSE flags, with three multipliers: random complex
with |m| in [0.5, 2), the spectral derivative i k_x, and m = 1 (which is the round trip).  The reference is a long-double
convolution (tests/ldfft.py, ld_r2c / ld_c2r of test_gpu_r2c.py) of the precision-rounded input and multiplier; there are two
transforms, so the bounds are twice those of a single one: rel_l2 <= 2.0 * eps * log2(Ntot), linf <= 8 * eps * log2(Ntot) relative
to rms(ref).  Outputs are NaN-prefilled and fenced with canaries.  Then full cubes against scipy fp64, the plan against the
three-call sequence it replaces (forward plan, torch multiply, backward plan), refilled inputs with new multipliers, in place,
compute-sanitizer, and P = 2, 4, 8 device-threads (skipped on a smaller box).  Each case prints "CONV-RATIO" lines."""
import faulthandler
import os
import sys
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from ld_harness import ratios64  # noqa: E402
from test_gpu_r2c import CANARY, CDT, EPS, RDT, fenced, ld_c2r, ld_r2c, need  # noqa: E402

K_L2, K_LINF = 2 * ldfft.REL_L2_K, 2 * ldfft.LINF_K
WORST = {}
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(autouse=True)
def _watchdog():
    faulthandler.dump_traceback_later(900, exit=True, file=sys.stderr)
    yield
    faulthandler.cancel_dump_traceback_later()


def check(got, ref, prec, ntot, what, fam):
    big = np.asarray(ref).dtype in (np.float64, np.complex128)
    rl2, linf = (ratios64 if big else ldfft.ratios)(got, ref, EPS[prec], ntot)
    print(f"CONV-RATIO {what} rel_l2 {rl2:.3f} linf {linf:.3f}")
    key = (fam, "fp64" if prec == dfft.DOUBLE else "fp32")
    WORST[key] = max(WORST.get(key, (0, 0)), (rl2, linf))
    assert rl2 <= K_L2 and linf <= K_LINF, (what, rl2, linf)


def rnd(shape, real, prec, seed):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(shape) if real else rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    return a.astype(RDT[prec][0] if real else CDT[prec][0])


def multipliers(n0, n1, h, prec, seed):
    rng = np.random.default_rng(seed)
    shape = (n0, n1, h)
    m_rand = rng.uniform(0.5, 2.0, shape) * np.exp(2j * np.pi * rng.uniform(size=shape))
    k = np.fft.fftfreq(n0, 1.0 / n0)
    m_dx = np.broadcast_to((1j * k)[:, None, None], shape)
    return {"rand": m_rand.astype(CDT[prec][0]), "dx": np.ascontiguousarray(m_dx).astype(CDT[prec][0]),
            "one": np.ones(shape, dtype=CDT[prec][0])}


def ld_forward(A, real):
    return ld_r2c(A) if real else ldfft.fftn(A)


def ld_inverse(S, M, real, n2):
    if real:
        return ld_c2r(S * M.astype(np.clongdouble), n2)
    return ldfft.fftn(S * M.astype(np.clongdouble), sign=1)


def ld_conv(A, M, real):
    return ld_inverse(ld_forward(A, real), M, real, A.shape[2])


def run_conv(A, mults, prec, real, flags=0, inplace=False, repeat=1):
    """one P = 1 convolve plan on fenced buffers; returns {name: output} (numpy, natural [x][y][z])"""
    torch.cuda.set_device(0)
    n0, n1, n2 = A.shape
    n = A.size
    tdt = RDT[prec][1] if real else CDT[prec][1]
    a_in, ilo, ihi = fenced(A.reshape(-1).copy(), tdt)
    inp = a_in[CANARY: CANARY + n]
    if inplace:
        a_out, lo, hi, out = a_in, ilo, ihi, inp
    else:
        a_out, lo, hi = fenced(n, tdt)
        out = a_out[CANARY: CANARY + n]
    plan = dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, inp.data_ptr(), None if inplace else out.data_ptr(), None, 0, 1, prec, flags, real=real)
    assert (plan.in_count, plan.out_count) == (n, n)
    res = {}
    for name, M in mults.items():
        m_t = torch.from_numpy(M.reshape(-1).copy()).cuda()
        first = None
        for _ in range(repeat):
            if inplace:
                out[:] = float("nan")
            plan.execute_convolve(m_t.data_ptr())
            plan.synchronize()
            cur = out.cpu().numpy().copy()
            assert first is None or np.array_equal(cur.view(np.uint8), first.view(np.uint8)), "executes differ"
            first = cur
        assert torch.equal(m_t.cpu(), torch.from_numpy(M.reshape(-1))), "multiplier changed"
        assert not np.isnan(first).any(), "unwritten output"
        res[name] = first.reshape(A.shape)
    t = plan.timings()
    assert len(t) == 5 and t[3] > 0 and abs(t[4] - (t[0] + t[2] + t[3])) < 1e-6
    plan.destroy()
    torch.cuda.synchronize()
    assert torch.equal(a_out[:CANARY], lo) and torch.equal(a_out[CANARY + n:], hi), "canary overwritten"
    if not inplace:
        assert torch.equal(inp.cpu(), torch.from_numpy(A.reshape(-1))), "input changed"
    return res


def tuned(prec):
    return [n for n in dfft.supported_lengths(prec) if dfft.length_kind(n, prec) == 2]


@pytest.mark.parametrize("real", [False, True], ids=["c2c", "r2c"])
@pytest.mark.parametrize("prec", [dfft.DOUBLE, dfft.FLOAT], ids=["fp64", "fp32"])
def test_every_tuned_x_length(prec, real):
    """thin slabs: (n1, n2) = (9, 10), and a generic y length (14) every other length; default and NO_TMA | NO_FUSE flags"""
    for i, n0 in enumerate(tuned(prec)):
        n1, n2 = (9, 10) if i % 2 == 0 else (14, 9)
        A = rnd((n0, n1, n2), real, prec, n0)
        h = n2 // 2 + 1 if real else n2
        mults = multipliers(n0, n1, h, prec, n0 + 1)
        S = ld_forward(A, real)
        refs = {k: ld_inverse(S, M, real, n2) for k, M in mults.items() if k != "one"}
        refs["one"] = A.astype(np.clongdouble) * A.size          # m = 1: the round trip, exact
        for flags in (0, dfft.NO_TMA | dfft.NO_FUSE):
            got = run_conv(A, mults, prec, real, flags, repeat=2 if flags == 0 else 1)
            for k in mults:
                check(got[k], refs[k], prec, A.size, f"{'r2c' if real else 'c2c'} n0={n0} {n1}x{n2} m={k} flags={flags}",
                      "thin-" + ("r2c" if real else "c2c"))


@pytest.mark.parametrize("prec", [dfft.DOUBLE, dfft.FLOAT], ids=["fp64", "fp32"])
def test_many_tiles_per_cta_scaled_and_in_place(prec):
    """n1 * ceil(n2 / C) tiles well beyond 3 per resident CTA; DFFT_SCALE_BACKWARD (m = 1 returns the input); in place"""
    for real in (False, True):
        n0, n1, n2 = 64, 200, 250 if not real else 243
        A = rnd((n0, n1, n2), real, prec, 5)
        h = n2 // 2 + 1 if real else n2
        mults = multipliers(n0, n1, h, prec, 6)
        got = run_conv(A, {"rand": mults["rand"], "one": mults["one"]}, prec, real, dfft.SCALE_BACKWARD, inplace=True)
        ref = ld_conv(A, mults["rand"], real) / A.size
        check(got["rand"], ref, prec, A.size, f"many-tiles scaled in-place {'r2c' if real else 'c2c'}", "many-tiles")
        check(got["one"], A, prec, A.size, f"many-tiles m=1 scaled {'r2c' if real else 'c2c'}", "many-tiles")


def sp_conv(A, M, real):
    import scipy.fft as sf
    A = A.astype(np.float64 if real else np.complex128)
    if real:
        return sf.irfftn(sf.rfftn(A, workers=-1) * M, s=A.shape, workers=-1) * A.size
    return sf.ifftn(sf.fftn(A, workers=-1) * M, workers=-1) * A.size


@pytest.mark.parametrize("n,prec,real", [(512, dfft.DOUBLE, False), (512, dfft.DOUBLE, True), (768, dfft.FLOAT, False)],
                         ids=["512-fp64-c2c", "512-fp64-r2c", "768-fp32-c2c"])
def test_full_cubes_against_scipy(n, prec, real):
    A = rnd((n, n, n), real, prec, 7)
    h = n // 2 + 1 if real else n
    M = multipliers(n, n, h, prec, 8)["rand"]
    got = run_conv(A, {"rand": M}, prec, real)["rand"]
    check(got, sp_conv(A, M, real), prec, A.size, f"cube {n}^3 {'r2c' if real else 'c2c'}", "cubes")


@pytest.mark.parametrize("prec", [dfft.DOUBLE, dfft.FLOAT], ids=["fp64", "fp32"])
def test_matches_the_three_call_sequence(prec):
    """forward C2C plan, torch multiply in the transposed spectrum layout, backward plan: the sequence the convolve plan replaces"""
    n = 256
    torch.cuda.set_device(0)
    A = rnd((n, n, n), False, prec, 9)
    M = multipliers(n, n, n, prec, 10)["rand"]
    got = run_conv(A, {"rand": M}, prec, False)["rand"]
    a = torch.from_numpy(A.reshape(-1)).cuda()
    spec = torch.empty_like(a)
    fwd = dfft.fft_mpi_plan_dft_c2c_3d(n, n, n, a.data_ptr(), spec.data_ptr(), None, 0, 1, dfft.FORWARD, prec)
    out = torch.empty_like(a)
    bwd = dfft.fft_mpi_plan_dft_c2c_3d(n, n, n, spec.data_ptr(), out.data_ptr(), None, 0, 1, dfft.BACKWARD, prec)
    mt = torch.from_numpy(np.ascontiguousarray(M.transpose(1, 2, 0)).reshape(-1)).cuda()   # [y][z][x], the spectrum's layout
    fwd.execute(); fwd.synchronize()
    prod = spec * mt
    torch.cuda.synchronize()
    dfft.lib().dfft_memcpy(bwd.bufferDev1, prod.data_ptr(), prod.numel() * prod.element_size(), 0)
    bwd.execute(); bwd.synchronize()
    seq = out.cpu().numpy().reshape(A.shape)
    fwd.destroy(); bwd.destroy()
    check(got, seq.astype(np.complex128), prec, A.size, "vs three-call sequence 256^3", "vs-sequence")


@pytest.mark.parametrize("real", [False, True], ids=["c2c", "r2c"])
def test_refilled_input_new_multiplier_each_execute(real):
    prec = dfft.DOUBLE
    n0, n1, n2 = 64, 40, 48
    torch.cuda.set_device(0)
    tdt = RDT[prec][1] if real else CDT[prec][1]
    n = n0 * n1 * n2
    a_out, lo, hi = fenced(n, tdt)
    out = a_out[CANARY: CANARY + n]
    inp = torch.zeros(n, dtype=tdt, device="cuda")
    plan = dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, inp.data_ptr(), out.data_ptr(), None, 0, 1, prec, 0, real=real)
    h = n2 // 2 + 1 if real else n2
    for k in range(3):
        A = rnd((n0, n1, n2), real, prec, 100 + k)
        M = multipliers(n0, n1, h, prec, 200 + k)["rand"]
        dfft.memcpy_htod(plan.bufferDev1, A.ctypes.data, A.nbytes)
        m_t = torch.from_numpy(M.reshape(-1).copy()).cuda()
        plan.execute_convolve(m_t.data_ptr())
        plan.synchronize()
        check(out.cpu().numpy().reshape(A.shape), ld_conv(A, M, real), prec, n, f"refill {k} {'r2c' if real else 'c2c'}", "refill")
    plan.destroy()
    torch.cuda.synchronize()
    assert torch.equal(a_out[:CANARY], lo) and torch.equal(a_out[CANARY + n:], hi)


@pytest.mark.parametrize("prec", [dfft.DOUBLE, dfft.FLOAT], ids=["fp64", "fp32"])
def test_compute_sanitizer_memcheck_and_racecheck(prec, tmp_path):
    import shutil
    import subprocess
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    script = tmp_path / "conv.py"
    script.write_text(
        "import sys; sys.path.insert(0, %r)\n"
        "import numpy as np, torch, distributedfft_b200 as dfft\n"
        "for real in (False, True):\n"
        "    n0, n1, n2 = 64, 12, 10\n"
        "    dt = (torch.float64 if %d == 0 else torch.float32) if real else (torch.complex128 if %d == 0 else torch.complex64)\n"
        "    cdt = torch.complex128 if %d == 0 else torch.complex64\n"
        "    a = torch.ones(n0 * n1 * n2, dtype=dt, device='cuda'); o = torch.empty_like(a)\n"
        "    m = torch.ones(n0 * n1 * (n2 // 2 + 1 if real else n2), dtype=cdt, device='cuda')\n"
        "    p = dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, a.data_ptr(), o.data_ptr(), None, 0, 1, %d, 0, real=real)\n"
        "    p.execute_convolve(m.data_ptr()); p.synchronize(); p.destroy()\n"
        "print('ok')\n" % (os.path.dirname(HERE), prec, prec, prec, prec))
    for tool in ("memcheck", "racecheck"):
        r = subprocess.run([cs, "--tool", tool, "--error-exitcode", "7", sys.executable, str(script)], capture_output=True, text=True, timeout=900)
        if "Error: Device not supported" in r.stdout or "SUMMARY" not in r.stdout:   # the tool could not attach here
            pytest.skip("compute-sanitizer cannot run on this device here: " + (r.stdout + r.stderr)[-300:])
        assert r.returncode == 0, (tool, r.stdout[-3000:], r.stderr[-2000:])
        assert "ERROR SUMMARY: 0 errors" in r.stdout or "RACECHECK SUMMARY: 0 hazards" in r.stdout, (tool, r.stdout[-1500:])


def run_multi(n0, n1, n2, P, A, M, flags, real):
    """P device-threads; returns the gathered natural-order output"""
    comm = dfft.LocalComm(P)
    xd, yd = -(-n0 // P), -(-n1 // P)
    tdt = RDT[dfft.DOUBLE][1] if real else CDT[dfft.DOUBLE][1]
    outs, errs = [None] * P, []

    def worker(p):
        try:
            torch.cuda.set_device(p)
            a = torch.from_numpy(A[p * xd: min(n0, (p + 1) * xd)].reshape(-1).copy()).to(tdt).cuda()
            o = torch.full_like(a, float("nan"))
            m = torch.from_numpy(np.ascontiguousarray(M[:, p * yd: min(n1, (p + 1) * yd)]).reshape(-1)).cuda()
            plan = dfft.fft_mpi_plan_dft_convolve_3d(n0, n1, n2, a.data_ptr(), o.data_ptr(), comm, p, P, dfft.DOUBLE, flags, real=real)
            for _ in range(3):
                plan.execute_convolve(m.data_ptr())
            plan.synchronize()
            outs[p] = o.cpu().numpy()
            plan.destroy()
        except Exception as e:  # pragma: no cover
            errs.append(repr(e))
    th = [threading.Thread(target=worker, args=(p,)) for p in range(P)]
    [t.start() for t in th]
    [t.join() for t in th]
    comm.destroy()
    assert not errs, errs
    return np.concatenate(outs).reshape(n0, n1, n2)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("P,n0,n1,n2", [(2, 64, 64, 64), (4, 64, 48, 40), (3, 100, 10, 9), (8, 256, 64, 32)])
@pytest.mark.parametrize("real", [False, True], ids=["c2c", "r2c"])
def test_multi_gpu(mode, P, n0, n1, n2, real):
    need(P)
    flags = dfft.EXCHANGE_P2P if mode == "p2p" else dfft.EXCHANGE_NCCL
    A = rnd((n0, n1, n2), real, dfft.DOUBLE, P)
    M = multipliers(n0, n1, n2 // 2 + 1 if real else n2, dfft.DOUBLE, P + 1)["rand"]
    got = run_multi(n0, n1, n2, P, A, M, flags, real)
    check(got, sp_conv(A, M, real), dfft.DOUBLE, A.size, f"P={P} {mode} {n0}x{n1}x{n2} {'r2c' if real else 'c2c'}", "multi")


def test_zz_report_worst_ratios():
    for (fam, prec), (rl2, linf) in sorted(WORST.items()):
        print(f"CONV-WORST {fam:14s} {prec} rel_l2 {rl2:.3f} linf {linf:.3f}")
