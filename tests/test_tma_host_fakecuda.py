"""CPU test of the host side of the TMA-pipelined passes: which passes a plan sends to the TMA kernels and the tensor maps it
encodes for them.  The library's objects are linked against tests/fakecuda/fake_cudart.cpp (as in
test_control_flow_fakecuda.py); with FAKECUDA_TMA=1 its cudaGetDriverEntryPoint hands out a stand-in cuTensorMapEncodeTiled that
enforces the driver's documented constraints (rank 3, 16-byte-aligned base, strides multiples of 16 bytes, box dims 1..256
and within their dims, inner box row a multiple of 16 bytes) and logs every map.  Plans are created and executed in a
subprocess, because the library looks the entry point up once per process.

Checked for every entry of tests/tma_entries.py and every mode, by default and under DFFT_TMA=2: the plan's tma_mask bits,
the fused forward t0, and the geometry of each map.  Y: dims (2*n2, n1, n0l), strides (n2, n1*n2) * element size, box
(2C, min(N, 256), 1).  X: dims (2*n2, n1l, n0), strides (n2, n1l*n2) * element size, box (2C, 1, min(N, 256)), including
P = 2 and P = 4 local-communicator plans with uneven splits -- the only check the X maps of multi-device splits get without
several GPUs.  Also: mixed-length plans under DFFT_TMA=2 (each axis keeps the entry of its own length), an existing plan is
unchanged by the creation of a plan of another length on the same thread, and a complex64 plan whose bufferDev2 is 8 bytes
off 16-byte alignment runs no TMA kernel (a complex128 one is rejected)."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

from test_control_flow_fakecuda import ROOT, fake_lib  # noqa: F401  (fixture)
from tma_entries import DOUBLE, ENTRIES, FLOAT, MASK_BIT, entry_id, esz, modes, rows, thin_shape

sys.path.insert(0, ROOT)
from oracle import SlabGeometry  # noqa: E402

WORKER = textwrap.dedent(r'''
    import ctypes, json, os, sys, threading
    sys.path.insert(0, sys.argv[1])
    import distributedfft_b200.api as api
    api.LIB_PATH = sys.argv[2]
    api._lib = None
    import distributedfft_b200 as dfft
    L = dfft.lib()
    L.fakecuda_tma_maps.restype = ctypes.c_longlong
    L.fakecuda_tma_maps.argtypes = [ctypes.c_void_p, ctypes.c_longlong]
    cases = json.loads(sys.argv[3])

    def maps():
        n = L.fakecuda_tma_maps(None, 0)
        buf = (ctypes.c_longlong * (11 * n))()
        L.fakecuda_tma_maps(buf, 11 * n)
        return [list(buf[11 * i: 11 * i + 11]) for i in range(n)]

    def alloc(count, prec):
        return dfft.fft_mpi_alloc_local_memory(count + 2, dfft.ALLOC_DEV, prec)   # room for an offset view

    def run(c):
        os.environ["DFFT_TMA"] = "2" if c["forced"] else "1"
        n0, n1, n2 = c["shape"]
        P, prec, off = c["P"], c["prec"], c.get("offset", 0)   # offset in bytes
        comm = dfft.LocalComm(P) if P > 1 else None
        out = {"masks": [None] * P, "fused": [None] * P, "errs": []}
        bufs = []
        L.fakecuda_tma_reset()
        def worker(p):
            try:
                mc = dfft.getMaxDataCount(n0, n1, n2, P, p == P - 1)
                a, b = alloc(mc, prec), alloc(mc, prec)
                bufs.append((a, b))
                if c["inplace"]:
                    src, dst = a + off, None
                else:
                    src, dst = a, b + off
                plan = dfft.fft_mpi_plan_dft_c2c_3d(n0, n1, n2, src, dst, comm, p, P, c["dir"], prec, c["flags"])
                out["masks"][p] = plan.tma_mask
                out["fused"][p] = plan.fused
                plan.execute(); plan.synchronize(); plan.destroy()
            except Exception as e:
                out["errs"].append(str(e))
        if P == 1:
            worker(0)
        else:
            th = [threading.Thread(target=worker, args=(p,)) for p in range(P)]
            [t.start() for t in th]; [t.join() for t in th]
        if comm: comm.destroy()
        for a, b in bufs:
            L.dfft_free_local(a, dfft.ALLOC_DEV); L.dfft_free_local(b, dfft.ALLOC_DEV)
        out["maps"] = maps()
        return out

    def two_plans(c):
        # plan A is created, then plan B of another length on the same thread; A executes after B's creation, then both alternately
        os.environ["DFFT_TMA"] = "2"
        res = {"maps": [], "masks": []}
        bufs, plans = [], []
        for shape in c["shapes"]:
            mc = dfft.getMaxDataCount(*shape, 1, True)
            a, b = alloc(mc, 0), alloc(mc, 0)
            bufs += [a, b]
            plans.append(dfft.fft_mpi_plan_dft_c2c_3d(*shape, a, b, None, 0, 1, dfft.FORWARD, 0, 0))
        for k in (0, 1, 0, 1):
            L.fakecuda_tma_reset()
            plans[k].execute(); plans[k].synchronize()
            res["maps"].append(maps()); res["masks"].append(plans[k].tma_mask)
        for p in plans: p.destroy()
        for a in bufs: L.dfft_free_local(a, dfft.ALLOC_DEV)
        return res

    results = [two_plans(c) if c.get("kind") == "two_plans" else run(c) for c in cases]
    print("RESULTS " + json.dumps(results))
''')

FWD, BWD = 1, -1
NO_PIPELINE, EXCHANGE_P2P, EXCHANGE_STAGED = 256, 1, 3


def _case(entry, shape, direction, forced, P=1, flags=0, inplace=False, offset=0, prec=None, **tags):
    return dict(shape=list(shape), dir=direction, forced=forced, P=P, flags=flags, inplace=inplace, offset=offset,
                prec=entry[1] if prec is None else prec, entry=list(entry[:3]), **tags)


def _y_map(prec, C, N, n0l, n1, n2):
    return [1, 8 if prec == DOUBLE else 7, 0, 2 * n2, n1, n0l, n2 * esz(prec), n1 * n2 * esz(prec), 2 * C, rows(N), 1]


def _x_map(prec, C, N, n0, n1l, n2):
    return [1, 8 if prec == DOUBLE else 7, 0, 2 * n2, n1l, n0, n2 * esz(prec), n1l * n2 * esz(prec), 2 * C, 1, rows(N)]


def _cases():
    cases = []
    for e in ENTRIES:
        N, prec, C, _ = e
        for forced in (False, True):
            used = modes(e, forced)
            for axis, mode_f, mode_b in ((2, "Z", "Z"), (1, "Y", "Y"), (0, "XF", "XB")):
                shape = thin_shape(e, axis)
                for d, mode in ((FWD, mode_f), (BWD, mode_b)):
                    n0, n1, n2 = shape
                    on = mode in used
                    want = []
                    if on and mode == "Y":
                        want = [_y_map(prec, C, N, n0, n1, n2)] * 2
                    elif on and mode in ("XF", "XB"):
                        want = [_x_map(prec, C, N, n0, n1, n2)]
                    cases.append(_case(e, shape, d, forced, mask=[MASK_BIT[mode] if on else 0], fused=[False], maps=want,
                                       what="%s %s %s" % (mode, "fwd" if d == FWD else "bwd", "forced" if forced else "default")))
            if "ZY" in e[3]:
                shape = (2, N, N)
                cases.append(_case(e, shape, FWD, forced, mask=[2 | (1 if forced else 0)], fused=[True], maps=[_y_map(prec, C, N, 2, N, N)],
                                   what="ZY forced" if forced else "ZY default"))
            # P = 2 and 4: uneven splits of n1 (and of n0 where N allows), X maps of every rank
            for P, n1 in ((2, 5), (4, 7)):
                shape = (N, n1, 16)
                g = SlabGeometry(N, n1, 16, P)
                xmaps = sorted(_x_map(prec, C, N, N, g.n1l(p), 16) for p in range(P))
                for d, flags, mode in ((FWD, EXCHANGE_P2P | NO_PIPELINE, "XF"), (FWD, EXCHANGE_STAGED, "XF"), (BWD, EXCHANGE_STAGED, "XB")):
                    on = mode in used
                    cases.append(_case(e, shape, d, forced, P=P, flags=flags, mask=[4 if on else 0] * P, fused=[False] * P, maps=xmaps if on else [],
                                       what="P=%d %s flags %d %s" % (P, mode, flags, "forced" if forced else "default")))
    # DFFT_TMA=2 on mixed-length fp64 shapes: every axis keeps its own entry
    by = {(e[0], e[1]): e for e in ENTRIES}
    z512, x1024, y512, y256, x512 = by[512, DOUBLE], by[1024, DOUBLE], by[512, DOUBLE], by[256, DOUBLE], by[512, DOUBLE]
    cases.append(_case(z512, (1024, 4, 512), FWD, True, mask=[1 | 4], fused=[False], maps=[_x_map(DOUBLE, 4, 1024, 1024, 4, 512)],
                       what="mixed Z512 X1024"))
    cases.append(_case(y512, (1024, 512, 8), FWD, True, mask=[2 | 4], fused=[False],
                       maps=[_y_map(DOUBLE, 8, 512, 1024, 512, 8)] * 2 + [_x_map(DOUBLE, 4, 1024, 1024, 512, 8)], what="mixed Y512 X1024"))
    cases.append(_case(y256, (512, 256, 16), FWD, True, mask=[2 | 4], fused=[False],
                       maps=[_y_map(DOUBLE, 16, 256, 512, 256, 16)] * 2 + [_x_map(DOUBLE, 8, 512, 512, 256, 16)], what="mixed Y256 X512"))
    # bufferDev2 at 8 mod 16: complex64 plans run no TMA kernel; out of place and in place, both directions
    f512 = by[512, FLOAT]
    for shape in (thin_shape(f512, 1), thin_shape(f512, 0), thin_shape(f512, 2)):
        for d in (FWD, BWD):
            for inplace in (False, True):
                cases.append(_case(f512, shape, d, False, inplace=inplace, offset=8, mask=[0], fused=[False], maps=[],
                                   what="misaligned fp32 %s" % ("in place" if inplace else "out of place")))
    cases.append(_case(by[1024, FLOAT], thin_shape(by[1024, FLOAT], 0), FWD, True, offset=8, mask=[0], fused=[False], maps=[],
                       what="misaligned fp32 forced"))
    for inplace in (False, True):
        cases.append(_case(y512, thin_shape(y512, 1), BWD, False, inplace=inplace, offset=8, error="16-byte aligned",
                           what="misaligned fp64"))
    return cases


def _run_worker(fake_lib, tmp_path, cases):
    script = tmp_path / "tma_worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, FAKECUDA_TMA="1")
    env.pop("DFFT_TMA", None)
    r = subprocess.run([sys.executable, str(script), ROOT, fake_lib, json.dumps(cases)], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [x for x in r.stdout.splitlines() if x.startswith("RESULTS ")]
    assert line, r.stdout[-3000:]
    return json.loads(line[-1][len("RESULTS "):])


def test_tma_masks_and_tensor_maps_of_every_entry_and_mode(fake_lib, tmp_path):
    cases = _cases()
    results = _run_worker(fake_lib, tmp_path, cases)
    bad = []
    covered = set()
    for c, r in zip(cases, results):
        tag = "%s %s shape %s: " % (entry_id(c["entry"]), c["what"], c["shape"])
        if "error" in c:
            if not any(c["error"] in e for e in r["errs"]):
                bad.append(tag + "expected an error containing %r, got %s" % (c["error"], r["errs"]))
            continue
        if r["errs"]:
            bad.append(tag + "failed: %s" % r["errs"])
            continue
        rejected = [m for m in r["maps"] if not m[0]]
        if rejected:
            bad.append(tag + "encode rejected %s" % rejected)
        if r["masks"] != c["mask"]:
            bad.append(tag + "tma_mask %s, want %s" % (r["masks"], c["mask"]))
        if r["fused"] != c["fused"]:
            bad.append(tag + "fused %s, want %s" % (r["fused"], c["fused"]))
        if sorted(r["maps"]) != sorted(c["maps"]):
            bad.append(tag + "maps %s, want %s" % (r["maps"], c["maps"]))
        if not any(b.startswith(tag) for b in bad) and c["mask"][0]:
            covered.add((tuple(c["entry"]), c["what"].split()[0] if c["P"] == 1 else "P", c["forced"]))
    assert not bad, "\n".join(bad)
    for e in ENTRIES:
        for forced in (False, True):
            for mode in modes(e, forced):
                assert (tuple(e[:3]), mode, forced) in covered, (e, mode, forced)


def test_an_existing_plan_keeps_its_entries_when_a_plan_of_another_length_is_created(fake_lib, tmp_path):
    # plan A: Y at 512 (C = 8); plan B, created after A on the same thread: X at 1024 (C = 4); DFFT_TMA=2
    cases = [dict(kind="two_plans", shapes=[[2, 512, 16], [1024, 2, 16]])]
    r = _run_worker(fake_lib, tmp_path, cases)[0]
    want_a = [_y_map(DOUBLE, 8, 512, 2, 512, 16)] * 2
    want_b = [_x_map(DOUBLE, 4, 1024, 1024, 2, 16)]
    assert r["masks"] == [2, 4, 2, 4]
    assert r["maps"] == [want_a, want_b, want_a, want_b]
