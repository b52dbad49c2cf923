"""Batched 2-D convolve lines plans (LinesConvolvePlan(two_d=...): dfft_lines_plan_create_convolve_2d / _r2c_2d) on the GPU.

The reference is a long-double 2-D convolution per image (tests/ldfft.py) of the precision-rounded input and multiplier.
There are two transforms, so the bounds are test_gpu_lines_conv.py's with Ntot = nx * ny: rel_l2 <= 2 * eps * log2(Ntot) and
max error / rms(ref) <= 8 * eps * log2(Ntot).  Cases:
- every instantiation of the one-kernel convolution (16, 32, 64 in fp64 and fp32, forced with DFFT_FORCE_PLANE=1 where the
  table leaves it off), shared and per-image multipliers, whole and partial groups of images per CTA;
- the pass path over every tuned ny, C2C and R2C, with even, odd and generic nx, scaled; large images;
- bitwise: the one-kernel convolution against DFFT_NO_PLANE=1 (the three passes) for all six instantiations, with more groups
  than resident CTAs; a shared multiplier against mult_count = batch with identical copies; in place against out of place;
- agreement with the three calls the plan replaces (LinesPlan / RealLinesPlan two_d forward, torch multiply, backward);
- fp32 at an odd complex64 offset, a refilled input with a new multiplier every execute;
- `in` and the multiplier unchanged, canaries around every buffer, three executes bitwise equal;
- compute-sanitizer memcheck / racecheck over the one-kernel convolution (skipped where the tool cannot attach).
Each case prints a "LINESCONV2D-RATIO" line."""
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

HERE = os.path.dirname(os.path.abspath(__file__))
DOUBLE, FLOAT = dfft.DOUBLE, dfft.FLOAT
K_L2, K_LINF = 2 * ldfft.REL_L2_K, 2 * ldfft.LINF_K
PLANE = (16, 32, 64)
# more groups of images than a 132-SM H100 holds resident CTAs (16: 4 images per CTA, 32: 2, 64: 1), with a partial last group
MANY = {16: 4227, 32: 1601, 64: 601}


@pytest.fixture(autouse=True)
def _watchdog(monkeypatch):
    faulthandler.dump_traceback_later(900, exit=True, file=sys.stderr)
    for var in ("DFFT_GENERIC", "DFFT_VARIANT", "DFFT_NO_PLANE", "DFFT_FORCE_PLANE"):
        monkeypatch.delenv(var, raising=False)
    yield
    faulthandler.cancel_dump_traceback_later()


def inputs(shape, prec, real, per_image, seed):
    """(a[batch][ny][nx], m): m is one image's multiplier, or [batch] of them; |m| in [0.5, 2), random phase"""
    nx, ny, batch = shape
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((batch, ny, nx))
    if not real:
        a = a + 1j * rng.standard_normal(a.shape)
    mshape = ((batch,) if per_image else ()) + (ny, nx // 2 + 1 if real else nx)
    m = rng.uniform(0.5, 2.0, mshape) * np.exp(2j * np.pi * rng.uniform(size=mshape))
    return a.astype(RDT[prec][0] if real else CDT[prec][0]), m.astype(CDT[prec][0])


def plan_ops(shape, prec, real, env):
    os.environ.pop("DFFT_NO_PLANE", None)
    os.environ.pop("DFFT_FORCE_PLANE", None)
    if env:
        os.environ[env] = "1"
    try:
        return [o["op"] for o in dfft.lines_conv_2d_ops(*shape, prec, real)]
    finally:
        os.environ.pop(env or "DFFT_NO_PLANE", None)


def run(shape, prec, a, m, real=False, flags=0, inplace=False, offset=0, env=None, repeat=3):
    """one plan on fenced buffers (env: DFFT_NO_PLANE or DFFT_FORCE_PLANE set at creation), executed `repeat` times from the
    same input; returns the output as numpy"""
    torch.cuda.set_device(0)
    batch = shape[2]
    if env:
        os.environ[env] = "1"
    try:
        plan = dfft.LinesConvolvePlan(two_d=shape, precision=prec, real=real, flags=flags)
    finally:
        if env:
            os.environ.pop(env)
    tdt = RDT[prec][1] if real else CDT[prec][1]
    flat, mflat = np.ascontiguousarray(a).reshape(-1), np.ascontiguousarray(m).reshape(-1)
    mc = batch if m.ndim == 3 else 1
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


def ld_conv2(a, m, real, scaled=False):
    """long-double ifft2(fft2(a) * m) * N (real: irfft2(rfft2(a) * m, s=(ny, nx)) * N) per image, N = nx * ny"""
    nx = a.shape[2]
    ml = m.astype(np.clongdouble)
    s = ldfft.fft(ldfft.fft(a.astype(np.clongdouble), 1), 2)
    if real:
        H = nx // 2 + 1
        y = ldfft.fft(s[:, :, :H] * ml, 1, +1)
        y[:, :, 0] = y[:, :, 0].real                  # what a C2R ignores: imaginary parts of x = 0 and x = nx/2
        if nx % 2 == 0:
            y[:, :, H - 1] = y[:, :, H - 1].real
        full = np.empty(a.shape, dtype=np.clongdouble)
        full[:, :, :H] = y
        full[:, :, H:] = np.conj(y[:, :, 1: nx - H + 1][:, :, ::-1])
        out = ldfft.fft(full, 2, +1).real
    else:
        out = ldfft.fft(ldfft.fft(s * ml, 2, +1), 1, +1)
    return out / (nx * a.shape[1]) if scaled else out


def check(got, ref, prec, what):
    ntot = int(np.prod(got.shape[1:]))
    rl2, linf = ldfft.ratios(got, ref, EPS[prec], ntot)
    print(f"LINESCONV2D-RATIO {what} rel_l2 {rl2:.3f} linf {linf:.3f}")
    assert rl2 <= K_L2 and linf <= K_LINF, (what, rl2, linf)


def same(x, y):
    return np.array_equal(x.view(np.uint8), y.view(np.uint8))


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
@pytest.mark.parametrize("n", PLANE)
def test_every_plane_conv_instantiation(n, prec):
    for batch in ({16: (1, 5, 8), 32: (3, 4), 64: (2,)}[n]):
        shape = (n, n, batch)
        assert plan_ops(shape, prec, False, "DFFT_FORCE_PLANE") == ["XY_PLANE_CONV"]
        for per_image in (False, True):
            for scaled in (False, True):
                a, m = inputs(shape, prec, False, per_image, seed=n + 7 * prec + 31 * batch + per_image + 2 * scaled)
                got = run(shape, prec, a, m, flags=dfft.SCALE_BACKWARD if scaled else 0, env="DFFT_FORCE_PLANE")
                check(got, ld_conv2(a, m, False, scaled), prec,
                      f"plane {shape} {PN[prec]} {'per-image' if per_image else 'shared'}{' scaled' if scaled else ''}")


def tuned(prec):
    return [n for n in dfft.supported_lengths(prec) if dfft.length_kind(n, prec) == 2]


@pytest.mark.parametrize("real", [False, True])
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_every_tuned_ny_on_the_pass_path(prec, real):
    nys = tuned(prec)
    assert len(nys) >= 10, nys
    for i, ny in enumerate(nys):
        nx = (12, 9, 14)[i % 3]                       # even, odd (generic for R2C) and generic nx
        shape = (nx, ny, 3)
        assert plan_ops(shape, prec, real, None) == (["Z_R2C", "XCONV", "Z_C2R"] if real else ["Z", "XCONV", "Z"])
        a, m = inputs(shape, prec, real, i % 2 == 1, seed=ny)
        got = run(shape, prec, a, m, real=real, flags=dfft.SCALE_BACKWARD, repeat=1)
        check(got, ld_conv2(a, m, real, scaled=True), prec, f"pass {'r2c' if real else 'c2c'} {shape} {PN[prec]}")


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_large_images(prec):
    cases = [((512, 512, 2), False), ((512, 512, 2), True), ((8, 4096, 5), False), ((10, 4096, 3), True), ((48, 48, 300), False)]
    if prec == FLOAT:
        cases += [((1024, 1024, 1), False), ((1024, 1024, 1), True)]
    for shape, real in cases:
        a, m = inputs(shape, prec, real, False, seed=sum(shape))
        got = run(shape, prec, a, m, real=real, repeat=1)
        check(got, ld_conv2(a, m, real), prec, f"large {'r2c' if real else 'c2c'} {shape} {PN[prec]}")


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_bitwise_identities(prec):
    """one-kernel convolution vs the three passes, shared vs identical per-image copies, in place vs out of place"""
    for n in PLANE:
        for batch in (MANY[n], 3):
            shape = (n, n, batch)
            a, m = inputs(shape, prec, False, False, seed=n + batch)
            base = run(shape, prec, a, m, env="DFFT_FORCE_PLANE", repeat=2)
            assert same(base, run(shape, prec, a, m, env="DFFT_NO_PLANE", repeat=1)), ("no-plane", shape)
            copies = np.ascontiguousarray(np.broadcast_to(m, (batch,) + m.shape))
            assert same(base, run(shape, prec, a, copies, env="DFFT_FORCE_PLANE", repeat=1)), ("per-image copies", shape)
            assert same(base, run(shape, prec, a, m, inplace=True, env="DFFT_FORCE_PLANE", repeat=1)), ("in place", shape)
            _, mb = inputs(shape, prec, False, True, seed=n + batch + 1)
            for flags in (0, dfft.SCALE_BACKWARD):
                assert same(run(shape, prec, a, mb, flags=flags, env="DFFT_FORCE_PLANE", repeat=1),
                            run(shape, prec, a, mb, flags=flags, env="DFFT_NO_PLANE", repeat=1)), ("per-image no-plane", shape, flags)
    for shape, real in (((12, 10, 4), False), ((16, 12, 3), True), ((64, 64, 2), True), ((48, 48, 5), False)):
        a, m = inputs(shape, prec, real, False, seed=5)
        base = run(shape, prec, a, m, real=real, repeat=1)
        copies = np.ascontiguousarray(np.broadcast_to(m, (shape[2],) + m.shape))
        assert same(base, run(shape, prec, a, copies, real=real, repeat=1)), shape
        assert same(base, run(shape, prec, a, m, real=real, inplace=True, repeat=1)), shape


def three_calls(shape, prec, a, m, real):
    """the sequence the plan replaces: forward 2-D lines plan, torch multiply, backward 2-D lines plan"""
    nx, ny, batch = shape
    mt = torch.from_numpy(np.ascontiguousarray(m)).cuda()
    if real:
        plan = dfft.RealLinesPlan(two_d=shape, precision=prec)
        x = torch.from_numpy(a.reshape(-1).copy()).cuda()
        s = torch.empty(batch * ny * (nx // 2 + 1), dtype=CDT[prec][1], device="cuda")
        torch.cuda.synchronize()
        plan.execute(x.data_ptr(), s.data_ptr(), dfft.FORWARD)
        plan.synchronize()
        s.view(batch, ny, -1).mul_(mt)
        torch.cuda.synchronize()
        plan.execute(s.data_ptr(), x.data_ptr(), dfft.BACKWARD)
    else:
        plan = dfft.LinesPlan(two_d=shape, precision=prec)
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
    for shape, real in (((32, 32, 9), False), ((64, 64, 4), False), ((20, 12, 3), False), ((64, 64, 4), True), ((15, 49, 3), True)):
        a, m = inputs(shape, prec, real, True, seed=3)
        got = run(shape, prec, a, m, real=real, repeat=1)
        torch.cuda.synchronize()
        check(got, three_calls(shape, prec, a, m, real), prec, f"vs three calls {'r2c' if real else 'c2c'} {shape} {PN[prec]}")


def test_fp32_at_an_odd_complex64_offset():
    for shape, env in (((32, 32, 3), "DFFT_FORCE_PLANE"), ((32, 32, 3), "DFFT_NO_PLANE"), ((12, 10, 2), None)):
        a, m = inputs(shape, FLOAT, False, False, seed=9)
        got = run(shape, FLOAT, a, m, offset=1, env=env)
        check(got, ld_conv2(a, m, False), FLOAT, f"offset {shape} f32 {env}")


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_refilled_input_and_new_multiplier_every_execute(prec):
    torch.cuda.set_device(0)
    for shape, real in (((16, 16, 5), False), ((64, 64, 3), False), ((12, 10, 3), True)):
        plan = dfft.LinesConvolvePlan(two_d=shape, precision=prec, real=real)
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
            plan.execute(x.data_ptr(), y.data_ptr(), mt.data_ptr(), shape[2] if it == 1 else 1)
            plan.synchronize()
            check(y.cpu().numpy().reshape(a.shape), ld_conv2(a, m, real), prec, f"refill {it} {shape} {PN[prec]}")
        plan.destroy()


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT])
def test_compute_sanitizer_memcheck_and_racecheck(prec, tmp_path):
    import shutil
    import subprocess
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    script = tmp_path / "lines_conv2d.py"
    script.write_text(
        "import sys; sys.path.insert(0, %r)\n"
        "import torch, distributedfft_b200 as dfft\n"
        "prec = %d\n"
        "cdt = torch.complex128 if prec == 0 else torch.complex64\n"
        "for n, batch in ((16, 5), (32, 3), (64, 2)):\n"
        "    a = torch.ones(n * n * batch, dtype=cdt, device='cuda'); o = torch.empty_like(a)\n"
        "    m = torch.ones(n * n * batch, dtype=cdt, device='cuda')\n"
        "    p = dfft.LinesConvolvePlan(two_d=(n, n, batch), precision=prec)\n"
        "    p.execute(a.data_ptr(), o.data_ptr(), m.data_ptr(), batch); p.execute(a.data_ptr(), a.data_ptr(), m.data_ptr(), 1)\n"
        "    p.synchronize(); p.destroy()\n"
        "print('ok')\n" % (os.path.dirname(HERE), prec))
    env = dict(os.environ, DFFT_FORCE_PLANE="1")
    for tool in ("memcheck", "racecheck"):
        r = subprocess.run([cs, "--tool", tool, "--error-exitcode", "7", sys.executable, str(script)], capture_output=True, text=True,
                           timeout=900, env=env)
        if "Error: Device not supported" in r.stdout or "SUMMARY" not in r.stdout:   # the tool could not attach here
            pytest.skip("compute-sanitizer cannot run on this device here: " + (r.stdout + r.stderr)[-300:])
        assert r.returncode == 0, (tool, r.stdout[-3000:], r.stderr[-2000:])
        assert "ERROR SUMMARY: 0 errors" in r.stdout or "RACECHECK SUMMARY: 0 hazards" in r.stdout, (tool, r.stdout[-1500:])
