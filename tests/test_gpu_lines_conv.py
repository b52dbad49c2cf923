"""Batched 3-D convolve lines plans (LinesConvolvePlan: dfft_lines_plan_create_convolve_3d / _r2c_3d) on the GPU.

The reference is a long-double convolution per volume (tests/ldfft.py; ld_r2c / ld_c2r of test_gpu_r2c.py) of the
precision-rounded input and multiplier.  There are two transforms, so the bounds are test_gpu_convolve.py's:
rel_l2 <= 2 * eps * log2(Ntot) and max error / rms(ref) <= 8 * eps * log2(Ntot), Ntot = nx * ny * nz.  Cases:
- every plane-kernel instantiation (16, 32, 64) in fp64 and fp32, C2C and R2C, shared and per-volume multipliers;
- non-plane shapes over every tuned nz from 4 to 128, C2C and R2C, scaled;
- bitwise: the plane kernel against DFFT_NO_PLANE=1, a shared multiplier against mult_count = batch with identical copies,
  in place against out of place;
- agreement with the three calls the plan replaces (LinesPlan forward, torch multiply, LinesPlan backward) within the bounds;
- fp32 at an odd complex64 offset, a refilled input with a new multiplier every execute;
- `in` and the multiplier unchanged, canaries around every buffer, three executes bitwise equal;
- compute-sanitizer memcheck / racecheck per precision (skipped where the tool cannot attach).
Each case prints a "LINESCONV-RATIO" line."""
import faulthandler
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from test_gpu_lines3d import CDT, EPS, PN, RDT, fenced  # noqa: E402
from test_gpu_r2c import ld_c2r, ld_r2c  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
DOUBLE, FLOAT = dfft.DOUBLE, dfft.FLOAT
K_L2, K_LINF = 2 * ldfft.REL_L2_K, 2 * ldfft.LINF_K
PLANE = (16, 32, 64)


@pytest.fixture(autouse=True)
def _watchdog(monkeypatch):
    faulthandler.dump_traceback_later(900, exit=True, file=sys.stderr)
    for var in ("DFFT_GENERIC", "DFFT_VARIANT", "DFFT_NO_PLANE", "DFFT_FORCE_PLANE"):
        monkeypatch.delenv(var, raising=False)
    yield
    faulthandler.cancel_dump_traceback_later()


def inputs(shape, prec, real, per_volume, seed):
    """(a[batch][nz][ny][nx], m): m is one volume's multiplier, or [batch] of them; |m| in [0.5, 2), random phase"""
    nx, ny, nz, batch = shape
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((batch, nz, ny, nx))
    if not real:
        a = a + 1j * rng.standard_normal(a.shape)
    mshape = ((batch,) if per_volume else ()) + (nz, ny, nx // 2 + 1 if real else nx)
    m = rng.uniform(0.5, 2.0, mshape) * np.exp(2j * np.pi * rng.uniform(size=mshape))
    return a.astype(RDT[prec][0] if real else CDT[prec][0]), m.astype(CDT[prec][0])


def run(shape, prec, a, m, real=False, flags=0, inplace=False, offset=0, no_plane=False, repeat=3):
    """one plan on fenced buffers, executed `repeat` times from the same input; returns the output as numpy"""
    torch.cuda.set_device(0)
    batch = shape[3]
    if no_plane:
        os.environ["DFFT_NO_PLANE"] = "1"
    try:
        plan = dfft.LinesConvolvePlan(shape, precision=prec, real=real, flags=flags)
    finally:
        os.environ.pop("DFFT_NO_PLANE", None)
    tdt = RDT[prec][1] if real else CDT[prec][1]
    flat, mflat = np.ascontiguousarray(a).reshape(-1), np.ascontiguousarray(m).reshape(-1)
    mc = batch if m.ndim == 4 else 1
    a_m, mult, mfence = fenced(mflat, CDT[prec][1], offset)
    try:
        first = None
        for _ in range(repeat):
            a_in, inp, ifence = fenced(flat, tdt, offset)
            if inplace:
                a_out, out, ofence = a_in, inp, ifence
            else:
                a_out, out, ofence = fenced(flat.size, tdt, offset)
            torch.cuda.synchronize()                 # the plan runs on its own stream
            plan.execute(inp.data_ptr(), out.data_ptr(), mult.data_ptr(), mc)
            plan.synchronize()
            cur = out.cpu().numpy().copy()
            for arena, view, (lo, hi) in ((a_out, out, ofence), (a_m, mult, mfence)) + (() if inplace else ((a_in, inp, ifence),)):
                k = lo.numel()
                assert torch.equal(arena[:k], lo) and torch.equal(arena[k + view.numel():], hi), "canary overwritten"
            if not inplace:
                assert torch.equal(inp.cpu(), torch.from_numpy(flat)), "input changed"
            assert torch.equal(mult.cpu(), torch.from_numpy(mflat)), "multiplier changed"
            if first is None:
                first = cur
            else:
                assert np.array_equal(cur.view(np.uint8), first.view(np.uint8)), "executes differ"
    finally:
        plan.destroy()
    assert not np.isnan(first.view(RDT[prec][0])).any(), "unwritten output"
    return first.reshape(a.shape)


def ld_conv(a, m, real, scaled=False):
    """long-double ifftn(fftn(a) * m) * N (real: irfftn(rfftn(a) * m) * N) per volume"""
    out = []
    for b in range(a.shape[0]):
        mb = (m[b] if m.ndim == 4 else m).astype(np.clongdouble)
        v = ld_c2r(ld_r2c(a[b]) * mb, a.shape[3]) if real else ldfft.fftn(ldfft.fftn(a[b]) * mb, sign=1)
        out.append(v / np.prod(a.shape[1:]) if scaled else v)
    return np.stack(out)


def check(got, ref, prec, what):
    ntot = int(np.prod(got.shape[1:]))
    rl2, linf = ldfft.ratios(got, ref, EPS[prec], ntot)
    print(f"LINESCONV-RATIO {what} rel_l2 {rl2:.3f} linf {linf:.3f}")
    assert rl2 <= K_L2 and linf <= K_LINF, (what, rl2, linf)


@pytest.mark.parametrize("real", [False, True])
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
@pytest.mark.parametrize("n", PLANE)
def test_every_plane_instantiation(n, prec, real):
    shape = {16: (16, 16, 16, 5), 32: (32, 32, 32, 3), 64: (64, 64, 64, 1)}[n]
    for per_volume in (False, True):
        a, m = inputs(shape, prec, real, per_volume, seed=n + 7 * prec + 31 * real + per_volume)
        got = run(shape, prec, a, m, real=real)
        check(got, ld_conv(a, m, real), prec, f"plane {'r2c' if real else 'c2c'} {shape} {PN[prec]} {'per-volume' if per_volume else 'shared'}")


def tuned_nz(prec):
    return [n for n in dfft.supported_lengths(prec) if dfft.length_kind(n, prec) == 2 and 4 <= n <= 128]


@pytest.mark.parametrize("real", [False, True])
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_every_tuned_nz_on_the_pass_path(prec, real):
    nzs = tuned_nz(prec)
    assert len(nzs) >= 10, nzs
    for i, nz in enumerate(nzs):
        shape = (12 if i % 2 else 9, 10, nz, 3)      # even and odd (generic for R2C) nx, a generic ny
        a, m = inputs(shape, prec, real, i % 2 == 1, seed=nz)
        got = run(shape, prec, a, m, real=real, flags=dfft.SCALE_BACKWARD, repeat=1)
        check(got, ld_conv(a, m, real, scaled=True), prec, f"pass {'r2c' if real else 'c2c'} {shape} {PN[prec]}")


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_bitwise_identities(prec):
    """plane kernel vs separate passes, shared vs identical per-volume copies, in place vs out of place"""
    for n in PLANE:
        shape = (n, n, 16, 6)
        a, m = inputs(shape, prec, False, False, seed=n)
        base = run(shape, prec, a, m)
        assert np.array_equal(base.view(np.uint8), run(shape, prec, a, m, no_plane=True).view(np.uint8)), ("no-plane", n)
        copies = np.ascontiguousarray(np.broadcast_to(m, (shape[3],) + m.shape))
        assert np.array_equal(base.view(np.uint8), run(shape, prec, a, copies).view(np.uint8)), ("per-volume copies", n)
        assert np.array_equal(base.view(np.uint8), run(shape, prec, a, m, inplace=True).view(np.uint8)), ("in place", n)
    for shape, real in (((12, 10, 32, 4), False), ((16, 12, 64, 3), True), ((64, 64, 16, 2), True)):
        a, m = inputs(shape, prec, real, False, seed=5)
        base = run(shape, prec, a, m, real=real)
        copies = np.ascontiguousarray(np.broadcast_to(m, (shape[3],) + m.shape))
        assert np.array_equal(base.view(np.uint8), run(shape, prec, a, copies, real=real).view(np.uint8)), shape
        assert np.array_equal(base.view(np.uint8), run(shape, prec, a, m, real=real, inplace=True).view(np.uint8)), shape


def three_calls(shape, prec, a, m, real):
    """the sequence the plan replaces: forward lines plan, torch multiply, backward lines plan"""
    nx, ny, nz, batch = shape
    mt = torch.from_numpy(np.ascontiguousarray(m)).cuda()
    if real:
        plan = dfft.RealLinesPlan(three_d=shape, precision=prec)
        x = torch.from_numpy(a.reshape(-1).copy()).cuda()
        s = torch.empty(batch * nz * ny * (nx // 2 + 1), dtype=CDT[prec][1], device="cuda")
        torch.cuda.synchronize()
        plan.execute(x.data_ptr(), s.data_ptr(), dfft.FORWARD)
        plan.synchronize()
        s.view(batch, nz, ny, -1).mul_(mt)
        torch.cuda.synchronize()
        plan.execute(s.data_ptr(), x.data_ptr(), dfft.BACKWARD)
    else:
        plan = dfft.LinesPlan(three_d=shape, precision=prec)
        x = torch.from_numpy(a.reshape(-1).copy()).cuda()
        torch.cuda.synchronize()
        plan.execute(x.data_ptr(), dfft.FORWARD)
        plan.synchronize()
        x.view(a.shape).mul_(mt)
        torch.cuda.synchronize()
        plan.execute(x.data_ptr(), dfft.BACKWARD)
    plan.synchronize()
    plan.destroy()
    return x.cpu().numpy().reshape(a.shape)


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_agrees_with_the_three_call_sequence(prec):
    for shape, real in (((32, 32, 32, 4), False), ((64, 64, 64, 2), False), ((20, 12, 48, 3), False), ((64, 64, 64, 2), True),
                        ((15, 14, 49, 3), True)):
        a, m = inputs(shape, prec, real, True, seed=3)
        got = run(shape, prec, a, m, real=real, repeat=1)
        torch.cuda.synchronize()
        check(got, three_calls(shape, prec, a, m, real), prec, f"vs three calls {'r2c' if real else 'c2c'} {shape} {PN[prec]}")


def test_fp32_at_an_odd_complex64_offset():
    for shape in ((32, 32, 32, 3), (12, 10, 16, 2)):
        a, m = inputs(shape, FLOAT, False, False, seed=9)
        got = run(shape, FLOAT, a, m, offset=1)
        check(got, ld_conv(a, m, False), FLOAT, f"offset {shape} f32")


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_refilled_input_and_new_multiplier_every_execute(prec):
    torch.cuda.set_device(0)
    for shape, real in (((16, 16, 16, 4), False), ((12, 10, 32, 3), True)):
        plan = dfft.LinesConvolvePlan(shape, precision=prec, real=real)
        tdt = RDT[prec][1] if real else CDT[prec][1]
        n = int(np.prod(shape))
        x = torch.empty(n, dtype=tdt, device="cuda")
        y = torch.empty(n, dtype=tdt, device="cuda")
        for it in range(3):
            a, m = inputs(shape, prec, real, it == 1, seed=100 + it)
            x.copy_(torch.from_numpy(a.reshape(-1)))
            mt = torch.from_numpy(m.reshape(-1).copy()).cuda()
            y.fill_(float("nan"))
            torch.cuda.synchronize()
            plan.execute(x.data_ptr(), y.data_ptr(), mt.data_ptr(), shape[3] if it == 1 else 1)
            plan.synchronize()
            check(y.cpu().numpy().reshape(a.shape), ld_conv(a, m, real), prec, f"refill {it} {shape} {PN[prec]}")
        plan.destroy()


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_compute_sanitizer_memcheck_and_racecheck(prec, tmp_path):
    import shutil
    import subprocess
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    script = tmp_path / "lines_conv.py"
    script.write_text(
        "import sys; sys.path.insert(0, %r)\n"
        "import torch, distributedfft_b200 as dfft\n"
        "prec = %d\n"
        "cdt = torch.complex128 if prec == 0 else torch.complex64\n"
        "for shape, real in (((16, 16, 16, 5), False), ((64, 64, 8, 1), False), ((12, 10, 16, 3), False), ((16, 16, 16, 3), True)):\n"
        "    nx, ny, nz, batch = shape\n"
        "    dt = (torch.float64 if prec == 0 else torch.float32) if real else cdt\n"
        "    a = torch.ones(nx * ny * nz * batch, dtype=dt, device='cuda'); o = torch.empty_like(a)\n"
        "    m = torch.ones(nz * ny * (nx // 2 + 1 if real else nx), dtype=cdt, device='cuda')\n"
        "    p = dfft.LinesConvolvePlan(shape, precision=prec, real=real)\n"
        "    p.execute(a.data_ptr(), o.data_ptr(), m.data_ptr(), 1); p.synchronize(); p.destroy()\n"
        "print('ok')\n" % (os.path.dirname(HERE), prec))
    for tool in ("memcheck", "racecheck"):
        r = subprocess.run([cs, "--tool", tool, "--error-exitcode", "7", sys.executable, str(script)], capture_output=True, text=True, timeout=900)
        if "Error: Device not supported" in r.stdout or "SUMMARY" not in r.stdout:   # the tool could not attach here
            pytest.skip("compute-sanitizer cannot run on this device here: " + (r.stdout + r.stderr)[-300:])
        assert r.returncode == 0, (tool, r.stdout[-3000:], r.stderr[-2000:])
        assert "ERROR SUMMARY: 0 errors" in r.stdout or "RACECHECK SUMMARY: 0 hazards" in r.stdout, (tool, r.stdout[-1500:])
