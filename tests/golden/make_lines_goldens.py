"""Writes the two goldens that pin the lines engine (the dfft_lines_* plans):

- tests/golden/lines_plan_ops.json: one SHA-256 per case of the JSON that one of the five host-only hooks
  (dfft_debug_lines_ops, dfft_debug_real_lines_ops, dfft_debug_lines_3d_ops, dfft_debug_lines_conv_3d_ops and
  dfft_debug_lines_conv_2d_ops) returns, or the hook's return code for a spec it rejects.  The cases cover both precisions and
  directions, tuned and run-time-scheduled lengths, four-step long lines, strided columns (dense, padded, gapped and
  interleaved; overlapping ones are rejected), square and non-square 2-D and 3-D
  plans with the plane kernels on, off (DFFT_NO_PLANE), forced (DFFT_FORCE_PLANE) and generic (DFFT_GENERIC), real plans,
  convolve plans (C2C and R2C, one or per-image multipliers, scaled or not) and odd batches, whose last tile or real pair is
  partial.
- tests/golden/lines_launch_traces.json: one SHA-256 per plan of the fake-runtime trace (fakecuda_trace) of create, a forward
  and a backward execute (convolve plans: executes with mult_count 1 and batch) and destroy, for every lines create entry
  point in both precisions.  It pins kernel identity, grid, block, shared memory and the event brackets, which the records of
  the hooks cannot see.

tests/test_lines_goldens.py checks that the library still returns exactly these.

    python tests/golden/make_lines_goldens.py [FAKE_LIB]              # rewrite both files
    python tests/golden/make_lines_goldens.py [FAKE_LIB] --show KEY   # print the records and traces of the cases whose key contains KEY

FAKE_LIB defaults to distributedfft_b200/build/libdfft_fakecuda.so, which the fakecuda tests build.  Regenerate only when a
lines schedule is meant to change, and say so in that change."""
import ctypes
import json
import os
import subprocess
import sys
import textwrap

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import distributedfft_b200 as dfft  # noqa: E402
from make_launch_traces import FAKE_LIB, digest  # noqa: E402

OPS_OUT = os.path.join(HERE, "lines_plan_ops.json")
TRACES_OUT = os.path.join(HERE, "lines_launch_traces.json")
# environment variables that change a lines schedule; cleared, then set per case
LINES_ENV = ("DFFT_NO_PLANE", "DFFT_FORCE_PLANE", "DFFT_GENERIC", "DFFT_NO_LONG_LINES", "DFFT_VARIANT")

DOUBLE, FLOAT, FORWARD, BACKWARD, SCALE_BACKWARD = dfft.DOUBLE, dfft.FLOAT, dfft.FORWARD, dfft.BACKWARD, dfft.SCALE_BACKWARD
PRECS = {"f64": DOUBLE, "f32": FLOAT}
DIRS = {"fwd": FORWARD, "bwd": BACKWARD}
ROWS = 1 << 31   # one more row than a plan takes


def ops_cases():
    """{key: (hook, args before (buf, cap), env)}"""
    out = {}

    def add(key, hook, args, env=None):
        assert key not in out, key
        out[key] = (hook, tuple(args), env or {})

    for pn, prec in PRECS.items():
        for dn, d in DIRS.items():
            s = "%s_%s" % (pn, dn)
            # complex 1-D: contiguous tuned and run-time-scheduled lengths over an odd line count, a four-step long line (built
            # whatever DFFT_NO_LONG_LINES says), strided columns; 2-D square and not
            for n in (16, 64, 128, 9, 14, 22, 360):
                add("lines_%d_x37_%s" % (n, s), "dfft_debug_lines_ops", (n, 1, 37, 37, n, 0, prec, d, 0))
            add("lines_64_x37_generic_%s" % s, "dfft_debug_lines_ops", (64, 1, 37, 37, 64, 0, prec, d, 0), {"DFFT_GENERIC": "1"})
            for n, lines in ((8192, 5), (65536, 3), (5 * 8192, 2)):
                add("lines_fourstep_%d_x%d_%s" % (n, lines, s), "dfft_debug_lines_ops", (n, 1, lines, lines, n, 0, prec, d, 0))
            add("lines_fourstep_8192_x5_nolong_%s" % s, "dfft_debug_lines_ops", (8192, 1, 5, 5, 8192, 0, prec, d, 0),
                {"DFFT_NO_LONG_LINES": "1"})
            add("lines_cols_96x21x3_%s" % s, "dfft_debug_lines_ops", (96, 21, 63, 21, 1, 96 * 21, prec, d, 0))
            add("lines_cols_64x10x3_%s" % s, "dfft_debug_lines_ops", (64, 10, 30, 10, 1, 640, prec, d, 0))
            # columns with padded rows, a gap between matrices, interleaved matrices
            add("lines_cols_padded_96x21x3_%s" % s, "dfft_debug_lines_ops", (96, 24, 63, 21, 1, 96 * 24, prec, d, 0))
            add("lines_cols_gapped_64x10x3_%s" % s, "dfft_debug_lines_ops", (64, 10, 30, 10, 1, 640 + 37, prec, d, 0))
            add("lines_cols_interleaved_48x7x2_%s" % s, "dfft_debug_lines_ops", (48, 14, 14, 7, 1, 7, prec, d, 0))
            for nx, ny, b in ((32, 32, 5), (64, 48, 3), (14, 22, 3), (16, 9, 1)):
                add("lines2d_%dx%dx%d_%s" % (nx, ny, b, s), "dfft_debug_lines_ops", (nx, ny, b, 0, 0, 0, prec, d, 1))
            # real 1-D and 2-D (odd line counts: a partial last pair)
            for n in (16, 64, 128, 9, 14, 22, 360):
                add("real_%d_x37_%s" % (n, s), "dfft_debug_real_lines_ops", (n, 1, 37, prec, d, 0))
            for nx, ny, b in ((64, 48, 3), (14, 10, 3), (32, 32, 5), (16, 9, 1)):
                add("real2d_%dx%dx%d_%s" % (nx, ny, b, s), "dfft_debug_real_lines_ops", (nx, ny, b, prec, d, 1))
            # 3-D: the plane kernel by default, off, forced and on generic entries; other shapes; real plans
            for n in (16, 32, 64):
                for en, env in (("", {}), ("_noplane", {"DFFT_NO_PLANE": "1"}), ("_forceplane", {"DFFT_FORCE_PLANE": "1"}),
                                ("_generic", {"DFFT_GENERIC": "1"})):
                    add("lines3d_%dx%dx4x3%s_%s" % (n, n, en, s), "dfft_debug_lines_3d_ops", (n, n, 4, 3, prec, d, 0), env)
            for sh in ((48, 48, 4, 2), (16, 8, 4, 3), (14, 22, 26, 1), (9, 9, 9, 2)):
                add("lines3d_%dx%dx%dx%d_%s" % (*sh, s), "dfft_debug_lines_3d_ops", (*sh, prec, d, 0))
            for sh in ((64, 64, 64, 1), (16, 16, 16, 3), (9, 8, 6, 3), (14, 12, 10, 2), (360, 6, 4, 1)):
                add("real3d_%dx%dx%dx%d_%s" % (*sh, s), "dfft_debug_lines_3d_ops", (*sh, prec, d, 1))
            add("real3d_16x16x16x3_generic_%s" % s, "dfft_debug_lines_3d_ops", (16, 16, 16, 3, prec, d, 1), {"DFFT_GENERIC": "1"})
        # convolve plans: C2C and R2C, mult_count 1 and batch, scaled or not, the plane-convolve sizes on, off and forced
        for real in (0, 1):
            rn = "r2c" if real else "c2c"
            for flags in (0, SCALE_BACKWARD):
                fn = "_scaled" if flags else ""
                for mc in (1, 3):
                    s = "%s_%s%s_m%d" % (pn, rn, fn, mc)
                    for sh in ((16, 16, 8, 3), (32, 32, 4, 3), (64, 64, 4, 3), (12, 10, 16, 3), (9, 8, 32, 3)):
                        add("conv3d_%dx%dx%dx%d_%s" % (*sh, s), "dfft_debug_lines_conv_3d_ops", (*sh, prec, real, flags, mc))
                    add("conv3d_16x16x8x3_noplane_%s" % s, "dfft_debug_lines_conv_3d_ops", (16, 16, 8, 3, prec, real, flags, mc),
                        {"DFFT_NO_PLANE": "1"})
                    for sh in ((16, 16, 3), (32, 32, 3), (64, 64, 3), (48, 32, 3), (14, 16, 3), (9, 64, 3)):
                        add("conv2d_%dx%dx%d_%s" % (*sh, s), "dfft_debug_lines_conv_2d_ops", (*sh, prec, real, flags, mc))
                    for n in (16, 32, 64):
                        for en, env in (("_noplane", {"DFFT_NO_PLANE": "1"}), ("_forceplane", {"DFFT_FORCE_PLANE": "1"})):
                            add("conv2d_%dx%dx3%s_%s" % (n, n, en, s), "dfft_debug_lines_conv_2d_ops", (n, n, 3, prec, real, flags, mc), env)
    # rejections: unsupported lengths and layouts, bad flags, directions and multiplier counts, more than 2^31 - 1 rows
    add("reject_lines_17_strided", "dfft_debug_lines_ops", (17, 4, 8, 4, 1, 68, DOUBLE, FORWARD, 0))
    add("reject_lines_prime_long", "dfft_debug_lines_ops", (8191, 1, 2, 2, 8191, 0, DOUBLE, FORWARD, 0))
    add("reject_lines_not_dense", "dfft_debug_lines_ops", (16, 1, 8, 4, 16, 80, DOUBLE, FORWARD, 0))
    add("reject_lines_fourstep_gapped", "dfft_debug_lines_ops", (8192, 1, 4, 2, 8192, 3 * 8192, DOUBLE, FORWARD, 0))
    # columns that overlap: more columns than a row holds, two matrices at one address, a negative matrix distance, interleaved
    # matrices that collide
    add("reject_lines_cols_overlap", "dfft_debug_lines_ops", (16, 4, 10, 5, 1, 80, DOUBLE, FORWARD, 0))
    add("reject_lines_cols_outer0", "dfft_debug_lines_ops", (16, 4, 8, 4, 1, 0, DOUBLE, FORWARD, 0))
    add("reject_lines_cols_outer_negative", "dfft_debug_lines_ops", (16, 4, 8, 4, 1, -64, DOUBLE, FORWARD, 0))
    add("reject_lines_cols_interleave_overlap", "dfft_debug_lines_ops", (16, 8, 8, 4, 1, 6, DOUBLE, FORWARD, 0))
    add("reject_real_17", "dfft_debug_real_lines_ops", (17, 1, 4, DOUBLE, FORWARD, 0))
    add("reject_real_1", "dfft_debug_real_lines_ops", (1, 1, 4, DOUBLE, FORWARD, 0))
    add("reject_real_direction", "dfft_debug_real_lines_ops", (16, 1, 4, DOUBLE, 0, 0))
    add("reject_real_rows", "dfft_debug_real_lines_ops", (16, 1 << 16, ROWS >> 16, DOUBLE, FORWARD, 1))
    add("reject_lines3d_17", "dfft_debug_lines_3d_ops", (17, 16, 16, 1, DOUBLE, FORWARD, 0))
    add("reject_lines3d_nz0", "dfft_debug_lines_3d_ops", (16, 16, 0, 1, DOUBLE, FORWARD, 0))
    add("reject_lines3d_direction", "dfft_debug_lines_3d_ops", (16, 16, 16, 1, DOUBLE, 2, 0))
    for real in (0, 1):
        add("reject_lines3d_rows_real%d" % real, "dfft_debug_lines_3d_ops", (16, 16, 16, ROWS >> 8, DOUBLE, FORWARD, real))
        add("reject_conv3d_rows_real%d" % real, "dfft_debug_lines_conv_3d_ops", (16, 16, 16, ROWS >> 8, DOUBLE, real, 0, 1))
        add("reject_conv2d_rows_real%d" % real, "dfft_debug_lines_conv_2d_ops", (16, 1 << 16, ROWS >> 16, DOUBLE, real, 0, 1))
        # a batch whose row count does not fit in 64 bits either
        add("reject_conv2d_rows_wrap_real%d" % real, "dfft_debug_lines_conv_2d_ops", (16, 16, 1 << 60, DOUBLE, real, 0, 1))
        add("reject_conv3d_rows_wrap_real%d" % real, "dfft_debug_lines_conv_3d_ops", (16, 16, 16, 1 << 60, DOUBLE, real, 0, 1))
        add("reject_conv3d_flag_real%d" % real, "dfft_debug_lines_conv_3d_ops", (16, 16, 16, 3, DOUBLE, real, SCALE_BACKWARD | 1, 1))
        add("reject_conv2d_flag_real%d" % real, "dfft_debug_lines_conv_2d_ops", (16, 16, 3, DOUBLE, real, SCALE_BACKWARD | 1, 1))
        add("reject_conv3d_nz14_real%d" % real, "dfft_debug_lines_conv_3d_ops", (16, 16, 14, 3, DOUBLE, real, 0, 1))
        add("reject_conv2d_ny14_real%d" % real, "dfft_debug_lines_conv_2d_ops", (16, 14, 3, DOUBLE, real, 0, 1))
        add("reject_conv2d_mult2_real%d" % real, "dfft_debug_lines_conv_2d_ops", (16, 16, 3, DOUBLE, real, 0, 2))
        add("reject_conv3d_generic_real%d" % real, "dfft_debug_lines_conv_3d_ops", (16, 16, 16, 3, DOUBLE, real, 0, 1),
            {"DFFT_GENERIC": "1"})
    return out


def hook_json(lib, hook, args, env):
    """the JSON text a hook returns for one case, or its return code (an int) when it rejects the spec"""
    for v in LINES_ENV:
        os.environ.pop(v, None)
    os.environ.update(env)
    try:
        fn = getattr(lib, hook)   # argument types as distributedfft_b200.api sets them
        need = fn(*args, None, 0)
        if need < 0:
            return int(need)
        buf = ctypes.create_string_buffer(int(need))
        fn(*args, buf, need)
        return buf.value.decode()
    finally:
        for v in env:
            os.environ.pop(v, None)


def plan_ops(keys=None):
    """{key: digest of the hook's JSON, or {"rc": code}} of every case (or of those in keys)"""
    lib = dfft.lib()
    out = {}
    for key, (hook, args, env) in ops_cases().items():
        if keys is not None and key not in keys:
            continue
        got = hook_json(lib, hook, args, env)
        out[key] = {"rc": got} if isinstance(got, int) else digest([got])
    return out


TRACE_WORKER = textwrap.dedent(r'''
    import ctypes, json, os, sys
    sys.path.insert(0, sys.argv[1])
    import distributedfft_b200.api as api
    api.LIB_PATH = sys.argv[2]
    api._lib = None
    import distributedfft_b200 as dfft
    L = dfft.lib()
    L.fakecuda_trace.restype = ctypes.c_longlong
    L.fakecuda_trace.argtypes = [ctypes.c_char_p, ctypes.c_longlong]
    L.fakecuda_live_allocations.restype = ctypes.c_longlong

    def trace():
        n = L.fakecuda_trace(None, 0)
        buf = ctypes.create_string_buffer(int(n))
        L.fakecuda_trace(buf, n)
        return buf.value.decode().splitlines()

    def alloc(nbytes):
        return dfft.fft_mpi_alloc_local_memory((nbytes + 15) // 16 + 1, dfft.ALLOC_DEV)

    def drive(make, run, nbytes, env):
        os.environ.update(env)
        bufs = [alloc(nbytes) for _ in range(3)]
        L.fakecuda_trace_reset()
        plan = make()
        run(plan, *bufs)
        plan.synchronize()
        plan.destroy()
        lines = trace()
        for b in bufs:
            L.dfft_free_local(b, dfft.ALLOC_DEV)
        for v in env:
            del os.environ[v]
        assert L.fakecuda_live_allocations() == 0, ("leak", L.fakecuda_live_allocations())
        return lines

    def c2c(plan, a, b, m):
        plan.execute(a, dfft.FORWARD); plan.execute(a, dfft.BACKWARD)

    def real(plan, a, b, m):
        plan.execute(a, b, dfft.FORWARD); plan.execute(b, a, dfft.BACKWARD)

    def conv(batch):
        return lambda plan, a, b, m: (plan.execute(a, b, m, 1), plan.execute(b, b, m, batch))

    result = {}
    noplane = {"DFFT_NO_PLANE": "1"}
    for pn, prec in (("f64", dfft.DOUBLE), ("f32", dfft.FLOAT)):
        def add(key, make, run, nbytes, env={}):
            result[key + "_" + pn] = drive(make, run, nbytes, env)
        for n, lines in ((64, 37), (22, 37), (8192, 5)):
            add("create_%d_x%d" % (n, lines), lambda: dfft.LinesPlan(n, 1, lines, lines, n, 0, prec), c2c, n * lines * 16)
        add("create_cols_96x21x3", lambda: dfft.LinesPlan(96, 21, 63, 21, 1, 96 * 21, prec), c2c, 96 * 63 * 16)
        for sh in ((64, 48, 3), (32, 32, 5)):
            add("create_2d_%dx%dx%d" % sh, lambda: dfft.LinesPlan(two_d=sh, precision=prec), c2c, sh[0] * sh[1] * sh[2] * 16)
        for sh, env in (((16, 16, 8, 3), {}), ((16, 16, 8, 3), noplane), ((48, 48, 4, 2), {}), ((14, 22, 26, 1), {})):
            add("create_3d_%dx%dx%dx%d%s" % (*sh, "_noplane" if env else ""), lambda: dfft.LinesPlan(three_d=sh, precision=prec), c2c,
                sh[0] * sh[1] * sh[2] * sh[3] * 16, env)
        for n, lines in ((64, 37), (22, 37)):
            add("create_r2c_%d_x%d" % (n, lines), lambda: dfft.RealLinesPlan(n, lines, prec), real, (n + 2) * lines * 16)
        add("create_r2c_2d_64x48x3", lambda: dfft.RealLinesPlan(two_d=(64, 48, 3), precision=prec), real, 66 * 48 * 3 * 16)
        for sh in ((16, 16, 16, 3), (9, 8, 6, 3)):
            add("create_r2c_3d_%dx%dx%dx%d" % sh, lambda: dfft.RealLinesPlan(three_d=sh, precision=prec), real,
                (sh[0] + 2) * sh[1] * sh[2] * sh[3] * 16)
        for sh, env in (((16, 16, 8, 3), {}), ((16, 16, 8, 3), noplane), ((12, 10, 16, 3), {})):
            add("create_convolve_3d_%dx%dx%dx%d%s" % (*sh, "_noplane" if env else ""),
                lambda: dfft.LinesConvolvePlan(three_d=sh, precision=prec), conv(sh[3]), sh[0] * sh[1] * sh[2] * sh[3] * 16, env)
        add("create_convolve_r2c_3d_16x16x16x3", lambda: dfft.LinesConvolvePlan(three_d=(16, 16, 16, 3), precision=prec, real=True,
            flags=dfft.SCALE_BACKWARD), conv(3), 18 * 16 * 16 * 3 * 16)
        for sh, env in (((32, 32, 5), {}), ((32, 32, 5), noplane), ((48, 32, 3), {})):
            add("create_convolve_2d_%dx%dx%d%s" % (*sh, "_noplane" if env else ""),
                lambda: dfft.LinesConvolvePlan(two_d=sh, precision=prec, flags=dfft.SCALE_BACKWARD), conv(sh[2]),
                sh[0] * sh[1] * sh[2] * 16, env)
        add("create_convolve_r2c_2d_16x16x5", lambda: dfft.LinesConvolvePlan(two_d=(16, 16, 5), precision=prec, real=True), conv(5),
            18 * 16 * 5 * 16)
    print(json.dumps(result))
''')


def launch_traces(fake_lib):
    """{plan key: trace lines} of every lines create entry point on the fake runtime"""
    env = {k: v for k, v in os.environ.items() if k not in LINES_ENV}
    r = subprocess.run([sys.executable, "-c", TRACE_WORKER, ROOT, fake_lib], capture_output=True, text=True, timeout=600, env=env)
    if r.returncode != 0:
        raise RuntimeError(r.stdout[-3000:] + r.stderr[-3000:])
    return json.loads(r.stdout.splitlines()[-1])


def main(argv):
    show = None
    if "--show" in argv:
        i = argv.index("--show")
        show = argv[i + 1]
        argv = argv[:i] + argv[i + 2:]
    lib = argv[0] if argv else FAKE_LIB
    traces = launch_traces(lib)
    if show is not None:
        for key, (hook, args, env) in ops_cases().items():
            if show in key:
                print("== %s" % key)
                print(hook_json(dfft.lib(), hook, args, env))
        for key, lines in traces.items():
            if show in key:
                print("== %s" % key)
                print("\n".join(lines))
        return
    ops = plan_ops()
    for path, out in ((OPS_OUT, ops), (TRACES_OUT, {k: digest(v) for k, v in traces.items()})):
        with open(path, "w") as f:
            json.dump(out, f, indent=0, sort_keys=True)
            f.write("\n")
        print("wrote", path, len(out), "cases")


if __name__ == "__main__":
    main(sys.argv[1:])
