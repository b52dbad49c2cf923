"""Batched 3-D lines plans (LinesPlan(three_d=...), RealLinesPlan(three_d=...)) and the plane kernel on the GPU.

Held to DESIGN section 4's bounds against the long-double FFT of tests/ldfft.py: rel_l2 <= 1.0 * eps * log2(Ntot) and
max error / rms(ref) <= 4 * eps * log2(Ntot), Ntot = nx * ny * nz.  Cases:
- every plane-kernel instantiation (16, 32, 64 in fp64 and fp32), forward and backward;
- the same with at least 3 plane groups per resident CTA, against scipy in fp64 (and at 64^3 x 64);
- bitwise equality of the default plan and the separate passes (DFFT_NO_PLANE=1), every instantiation, both directions,
  in place, several batch sizes -- the plane kernel runs the same schedules, twiddles and butterflies per line;
- non-square and generic shapes on the pass path; real plans with tuned, generic and odd nx (non-Hermitian C2R input);
- fp32 data at an odd complex64 offset (8-byte alignment) on the plane kernel;
- every buffer canary-fenced, real outputs NaN-prefilled, three executes bitwise equal;
- the batchFFT driver's 3d mode, compute-sanitizer memcheck / racecheck over the six plane kernels (skipped where the tool
  cannot attach), and the worst ratios per family on "LINES3D-RATIO" lines."""
import faulthandler
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import distributedfft_b200 as dfft  # noqa: E402
import ldfft  # noqa: E402
from ld_harness import ratios64  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
DOUBLE, FLOAT = dfft.DOUBLE, dfft.FLOAT
FWD, BWD = dfft.FORWARD, dfft.BACKWARD
RDT = {DOUBLE: (np.float64, torch.float64), FLOAT: (np.float32, torch.float32)}
CDT = {DOUBLE: (np.complex128, torch.complex128), FLOAT: (np.complex64, torch.complex64)}
EPS = {DOUBLE: ldfft.EPS["double"], FLOAT: ldfft.EPS["float"]}
PN = {DOUBLE: "f64", FLOAT: "f32"}
CANARY = 64
WORST = {}
PLANE = (16, 32, 64)
# shapes with >= 3 groups of planes per resident CTA on a 132-SM H100 (16: 4 planes per CTA, 32: 2, 64: 1)
MANY = {16: (16, 900), 32: (32, 120), 64: (64, 14)}


@pytest.fixture(autouse=True)
def _watchdog(monkeypatch):
    faulthandler.dump_traceback_later(600, exit=True, file=sys.stderr)
    for var in ("DFFT_GENERIC", "DFFT_VARIANT", "DFFT_NO_PLANE", "DFFT_FORCE_PLANE"):
        monkeypatch.delenv(var, raising=False)
    yield
    faulthandler.cancel_dump_traceback_later()


def fenced(host, tdt, offset=0):
    """device arena [canary | offset | data | canary]; `host` is flat numpy, or an int length for a NaN-filled buffer"""
    d = torch.device("cuda", 0)
    n = host if isinstance(host, int) else host.size
    rng = np.random.default_rng(99)
    pat = rng.standard_normal(2 * CANARY) if not tdt.is_complex else rng.standard_normal(2 * CANARY) + 1j * rng.standard_normal(2 * CANARY)
    pat = torch.from_numpy(pat).to(tdt).to(d)
    lo = CANARY + offset
    arena = torch.zeros(lo + n + CANARY, dtype=tdt, device=d)
    arena[:CANARY], arena[lo + n:] = pat[:CANARY], pat[CANARY:]
    if isinstance(host, int):
        arena[lo: lo + n] = float("nan")
    else:
        arena[lo: lo + n] = torch.from_numpy(host).to(d)
    return arena, arena[lo: lo + n], (arena[:lo].clone(), arena[lo + n:].clone())


def run_c2c(shape, prec, direction, host, offset=0, repeat=3, no_plane=False):
    """one in-place LinesPlan(three_d=shape) on a fenced copy of `host` (a[batch][nz][ny][nx]), executed `repeat` times from
    the same input; returns the output as numpy"""
    torch.cuda.set_device(0)
    if no_plane:
        os.environ["DFFT_NO_PLANE"] = "1"
    try:
        plan = dfft.LinesPlan(three_d=shape, precision=prec)
    finally:
        os.environ.pop("DFFT_NO_PLANE", None)
    flat = np.ascontiguousarray(host, dtype=CDT[prec][0]).reshape(-1)
    try:
        first = None
        for _ in range(repeat):
            arena, data, (lo, hi) = fenced(flat, CDT[prec][1], offset)
            plan.execute(data.data_ptr(), direction)
            plan.synchronize()
            cur = data.cpu().numpy().copy()
            k = lo.numel()
            assert torch.equal(arena[:k], lo) and torch.equal(arena[k + flat.size:], hi), "canary overwritten"
            if first is None:
                first = cur
            else:
                assert np.array_equal(cur.view(np.uint8), first.view(np.uint8)), "executes differ"
    finally:
        plan.destroy()
    assert not np.isnan(first.view(RDT[prec][0])).any()
    return first.reshape(np.shape(host))


def run_real(shape, prec, direction, host, repeat=3):
    nx, ny, nz, batch = shape
    rows = ny * nz * batch
    rc, cc = rows * nx, rows * (nx // 2 + 1)
    fwd = direction == FWD
    in_t, out_t = (RDT[prec][1], CDT[prec][1]) if fwd else (CDT[prec][1], RDT[prec][1])
    n_out = cc if fwd else rc
    flat = np.ascontiguousarray(host).reshape(-1)
    _, inp, _ = fenced(flat, in_t)
    a_out, out, (lo, hi) = fenced(n_out, out_t)
    plan = dfft.RealLinesPlan(three_d=shape, precision=prec)
    try:
        first = None
        for _ in range(repeat):
            plan.execute(inp.data_ptr(), out.data_ptr(), direction)
            plan.synchronize()
            cur = out.cpu().numpy().copy()
            if first is None:
                first = cur
            else:
                assert np.array_equal(cur.view(np.uint8), first.view(np.uint8)), "executes differ"
    finally:
        plan.destroy()
    torch.cuda.synchronize()
    assert torch.equal(a_out[:CANARY], lo) and torch.equal(a_out[CANARY + n_out:], hi), "canary overwritten"
    assert torch.equal(inp.cpu(), torch.from_numpy(flat)), "input changed"
    assert not np.isnan(first.view(RDT[prec][0])).any(), "unwritten output"
    return first


# ---- references ------------------------------------------------------------------------------------------------------------
def ld_fft3(a, sign):
    y = np.asarray(a).astype(np.clongdouble)
    for ax in (-1, -2, -3):
        y = ldfft.fft(y, ax, sign)
    return y


def ld_irfft3(S, nx):
    """numpy.fft.irfftn(S, s=(nz, ny, nx), axes=(1, 2, 3)) * nx*ny*nz with the imaginary parts of bin 0 and (even nx) nx/2
    dropped after the nz and ny inverses, as the C2R pass drops them"""
    y = S.astype(np.clongdouble)
    y = ldfft.fft(ldfft.fft(y, -3, +1), -2, +1)
    H = nx // 2 + 1
    y[..., 0] = y[..., 0].real
    if nx % 2 == 0:
        y[..., H - 1] = y[..., H - 1].real
    full = np.empty(y.shape[:-1] + (nx,), dtype=np.clongdouble)
    full[..., :H] = y
    full[..., H:] = np.conj(y[..., 1: nx - H + 1][..., ::-1])
    return ldfft.fft(full, -1, +1).real


def check(family, prec, got, ref, ntot, label, big=False):
    rl2, linf = (ratios64 if big else ldfft.ratios)(np.asarray(got).reshape(-1), np.asarray(ref).reshape(-1), EPS[prec], ntot)
    print("LINES3D-RATIO %-10s %-44s rel_l2 %6.3f  linf %6.3f" % (family, label, rl2, linf))
    w = WORST.get((family, prec), (0.0, 0.0))
    WORST[family, prec] = (max(w[0], rl2), max(w[1], linf))
    assert rl2 <= ldfft.REL_L2_K and linf <= ldfft.LINF_K, (label, rl2, linf)


def cdata(shape, prec, seed):
    nx, ny, nz, batch = shape
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((batch, nz, ny, nx)) + 1j * rng.standard_normal((batch, nz, ny, nx))).astype(CDT[prec][0])


# ---- the plane kernel --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", PLANE)
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
def test_plane_instantiations_against_long_double(n, prec):
    shape = (n, n, 6, 3)
    assert [o["op"] for o in dfft.lines_3d_ops(*shape, FWD, prec)] == ["XY_PLANE", "Y"]
    a = cdata(shape, prec, n)
    check("plane", prec, run_c2c(shape, prec, FWD, a), ld_fft3(a, -1), n * n * 6, f"fwd {n}^2x6x3 {PN[prec]}")
    check("plane", prec, run_c2c(shape, prec, BWD, a), ld_fft3(a, +1), n * n * 6, f"bwd {n}^2x6x3 {PN[prec]}")


@pytest.mark.parametrize("n", PLANE)
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
def test_plane_many_groups_per_cta_bitwise_and_against_scipy(n, prec):
    import scipy.fft
    nz, batch = MANY[n]
    shape = (n, n, nz, batch)
    a = cdata(shape, prec, 7 * n)
    for direction in (FWD, BWD):
        got = run_c2c(shape, prec, direction, a, repeat=2)
        ref = run_c2c(shape, prec, direction, a, repeat=1, no_plane=True)
        assert np.array_equal(got.view(np.uint8), ref.view(np.uint8)), ("plane kernel differs from the separate passes", n, direction)
        want = scipy.fft.fftn(a.astype(np.complex128), axes=(1, 2, 3)) if direction == FWD else \
            scipy.fft.ifftn(a.astype(np.complex128), axes=(1, 2, 3)) * (n * n * nz)
        check("plane-many", prec, got, want, n * n * nz, f"{'fwd' if direction == FWD else 'bwd'} {n}^2x{nz}x{batch} {PN[prec]}", big=True)


def test_64_cubed_x64_against_scipy():
    import scipy.fft
    shape = (64, 64, 64, 64)
    a = cdata(shape, DOUBLE, 6464)
    got = run_c2c(shape, DOUBLE, FWD, a, repeat=1)
    check("scipy", DOUBLE, got, scipy.fft.fftn(a, axes=(1, 2, 3)), 64 ** 3, "fwd 64^3x64 f64", big=True)
    got = run_c2c(shape, DOUBLE, BWD, a, repeat=1)
    check("scipy", DOUBLE, got, scipy.fft.ifftn(a, axes=(1, 2, 3)) * 64 ** 3, 64 ** 3, "bwd 64^3x64 f64", big=True)


@pytest.mark.parametrize("n", PLANE)
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
@pytest.mark.parametrize("nz,batch", [(2, 1), (5, 7), (3, 61)])
def test_plane_kernel_bitwise_equals_separate_passes(n, prec, nz, batch):
    shape = (n, n, nz, batch)
    a = cdata(shape, prec, n + nz + batch)
    for direction in (FWD, BWD):
        got = run_c2c(shape, prec, direction, a)
        ref = run_c2c(shape, prec, direction, a, no_plane=True)
        assert np.array_equal(got.view(np.uint8), ref.view(np.uint8)), (shape, direction)


@pytest.mark.parametrize("n", PLANE)
def test_plane_kernel_fp32_at_odd_complex64_offset(n):
    shape = (n, n, 4, 3)
    a = cdata(shape, FLOAT, 3 * n)
    got = run_c2c(shape, FLOAT, FWD, a, offset=1)
    check("offset", FLOAT, got, ld_fft3(a, -1), n * n * 4, f"fwd {n}^2x4x3 f32 +8 B")
    ref = run_c2c(shape, FLOAT, FWD, a, offset=1, no_plane=True)
    assert np.array_equal(got.view(np.uint8), ref.view(np.uint8))


# ---- the pass path -----------------------------------------------------------------------------------------------------------
# non-square, other tuned lengths, generic (14, 22, 26), odd (9, 125, 21), mixed radix (48, 12)
PASS_SHAPES = [(16, 8, 12, 3), (8, 32, 4, 5), (48, 48, 8, 2), (128, 128, 4, 1), (14, 22, 26, 1), (9, 9, 9, 5), (125, 6, 5, 2),
               (21, 10, 12, 3), (12, 48, 7, 1)]


@pytest.mark.parametrize("shape", PASS_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
def test_pass_path_shapes_against_long_double(shape, prec):
    assert all(o["op"] != "XY_PLANE" for o in dfft.lines_3d_ops(*shape, FWD, prec))
    nx, ny, nz, _ = shape
    a = cdata(shape, prec, sum(shape))
    check("passes", prec, run_c2c(shape, prec, FWD, a), ld_fft3(a, -1), nx * ny * nz, f"fwd {shape} {PN[prec]}")
    check("passes", prec, run_c2c(shape, prec, BWD, a), ld_fft3(a, +1), nx * ny * nz, f"bwd {shape} {PN[prec]}")


# ---- real plans --------------------------------------------------------------------------------------------------------------
REAL_SHAPES = [(64, 16, 8, 3), (32, 32, 32, 2), (14, 12, 10, 2), (9, 8, 6, 3), (125, 6, 4, 1), (360, 6, 4, 1)]


@pytest.mark.parametrize("shape", REAL_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
def test_real_plans_against_long_double(shape, prec):
    nx, ny, nz, batch = shape
    H = nx // 2 + 1
    rng = np.random.default_rng(sum(shape) * 3)
    x = rng.standard_normal((batch, nz, ny, nx)).astype(RDT[prec][0])
    got = run_real(shape, prec, FWD, x)
    check("real", prec, got, ld_fft3(x, -1)[..., :H], nx * ny * nz, f"r2c {shape} {PN[prec]}")
    S = (rng.standard_normal((batch, nz, ny, H)) + 1j * rng.standard_normal((batch, nz, ny, H))).astype(CDT[prec][0])
    got = run_real(shape, prec, BWD, S)
    check("real", prec, got, ld_irfft3(S, nx), nx * ny * nz, f"c2r {shape} {PN[prec]}")


# ---- driver, sanitizer, report -------------------------------------------------------------------------------------------------
def test_batch_driver_3d_mode(tmp_path):
    import re
    import subprocess
    exe = os.path.join(os.path.dirname(HERE), "distributedfft_b200", "batchFFT")
    assert os.path.exists(exe), "batchFFT was not built"
    csv = tmp_path / "batch_3d.csv"
    r = subprocess.run([exe, "3d", "64", "64", "64", "3", "1", str(csv)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "1 - FFT + iFFT C2C 3D in double precision LUT" in r.stdout
    m = re.search(r"FFT: (\S+) Buffer: ([0-9.]+) MB avg_hip_time: ([0-9.]+) ms Gflops: ([0-9.]+) num_iter: 3", r.stdout)
    assert m and m.group(1) == "64x64x64x256" and float(m.group(2)) == 1024.0, r.stdout
    err = float(re.search(r"Max error: (\S+)", r.stdout).group(1))
    assert err < 1e-6
    assert "element 0 input:  (1,0)" in r.stdout
    cols = csv.read_text().strip().split(",")
    assert len(cols) == 9 and cols[0] == "64"


@pytest.mark.parametrize("prec", [DOUBLE, FLOAT], ids=["fp64", "fp32"])
def test_compute_sanitizer_memcheck_and_racecheck(prec, tmp_path):
    import shutil
    import subprocess
    cs = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(cs):
        pytest.skip("compute-sanitizer not installed")
    script = tmp_path / "lines3d.py"
    script.write_text(
        "import sys; sys.path.insert(0, %r)\n"
        "import torch, distributedfft_b200 as dfft\n"
        "prec = %d\n"
        "cdt, rdt = (torch.complex128, torch.float64) if prec == 0 else (torch.complex64, torch.float32)\n"
        "for n in (16, 32, 64):\n"
        "    a = torch.ones(n * n * 3 * 3, dtype=cdt, device='cuda')\n"
        "    p = dfft.LinesPlan(three_d=(n, n, 3, 3), precision=prec)\n"
        "    p.execute(a.data_ptr(), 1); p.execute(a.data_ptr(), -1); p.synchronize(); p.destroy()\n"
        "r = torch.ones(16 * 12 * 5 * 2, dtype=rdt, device='cuda'); c = torch.ones(9 * 12 * 5 * 2, dtype=cdt, device='cuda')\n"
        "p = dfft.RealLinesPlan(three_d=(16, 12, 5, 2), precision=prec)\n"
        "p.execute(r.data_ptr(), c.data_ptr(), 1); p.execute(c.data_ptr(), r.data_ptr(), -1); p.synchronize(); p.destroy()\n"
        "print('ok')\n" % (os.path.dirname(HERE), prec))
    for tool in ("memcheck", "racecheck"):
        r = subprocess.run([cs, "--tool", tool, "--error-exitcode", "7", sys.executable, str(script)], capture_output=True, text=True, timeout=900)
        if "Error: Device not supported" in r.stdout or "SUMMARY" not in r.stdout:   # the tool could not attach here
            pytest.skip("compute-sanitizer cannot run on this device here: " + (r.stdout + r.stderr)[-300:])
        assert r.returncode == 0, (tool, r.stdout[-3000:], r.stderr[-2000:])
        assert "ERROR SUMMARY: 0 errors" in r.stdout or "RACECHECK SUMMARY: 0 hazards" in r.stdout, (tool, r.stdout[-1500:])


def test_zz_report_worst_ratios():
    for (family, prec), (rl2, linf) in sorted(WORST.items()):
        print("LINES3D-RATIO worst %-10s %s rel_l2 %6.3f  linf %6.3f" % (family, PN[prec], rl2, linf))
