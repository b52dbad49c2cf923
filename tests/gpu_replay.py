"""Replay of the multi-device schedules on ONE device, pass by pass.

A DFFT_DRY_RUN plan records every pass it would launch (tests/test_dry_run.py interprets the records with numpy).  Here the
records of the P per-device plans are launched on real kernels instead, one record at a time through the test hook
dfft_debug_launch_op, in the order the numpy interpreters run them (test_dry_run.schedule): per phase, the passes of every
virtual device, then that phase's all-to-alls as plain device-to-device copies.  Nothing runs concurrently and no kernel
waits on a flag, so the peer-store kinds (Y_CO, XB_CO, XCONV_CO, the fused t0 with the chunked store) and the chunked
loads (Y_CI, the fused inverse t0) run on one GPU exactly as addressed by a P-device plan: a peer's receive buffer is just
another allocation.

Every (virtual device, buffer) the records name gets its own allocation: NaN-prefilled, the caller's initial contents at the
start, random canaries before and after.  Before anything is launched, the footprint checker of test_dry_run_full_size walks
the same records on the CPU (every address inside its buffer, no element stored twice by a pass, no read of an element nobody
wrote), so a mapping mistake fails as a Python assertion instead of a stray device access.  Afterwards the canaries are checked
and so are the buffers that no record may write (bufferDev1, the multiplier, an out-of-place user input)."""
import numpy as np

import distributedfft_b200 as dfft
from test_dry_run import BUF1, IN, schedule
from test_dry_run_full_size import Footprints, boxes, mark, walk

CANARY = 48
MULT = 8          # the multiplier of a convolve plan (test_convolve_dry_run.MULT)
FUSED = ("fusedZ", "fusedY")
KEEP = (BUF1, MULT)   # buffers no record writes
NPDT = {dfft.DOUBLE: np.complex128, dfft.FLOAT: np.complex64}
ESZ = {dfft.DOUBLE: 16, dfft.FLOAT: 8}


class TorchMemory:
    """device memory of GPU 0 through torch"""

    def __init__(self):
        import torch
        self.torch = torch
        torch.cuda.set_device(0)

    def alloc(self, host):
        t = self.torch.from_numpy(host).to("cuda:0")
        return t, t.data_ptr()

    def fetch(self, t):
        self.torch.cuda.synchronize()
        return t.cpu().numpy()


class HostMemory:
    """host arrays: the memory of a fake CUDA runtime whose device memory is host memory"""

    def alloc(self, host):
        a = host.copy()
        return a, a.ctypes.data

    def fetch(self, a):
        return a


def launch_units(ops, nphases):
    """(device, record, second record or None) in schedule order: the two records of a fused t0 are one launch"""
    pending = None
    for d, op in schedule(ops, nphases):
        if pending is not None:
            pd, first = pending
            assert pd == d and first["phase"] == op["phase"] and op["op"] in FUSED and op["op"] != first["op"], (first["op"], op["op"])
            pending = None
            yield d, first, op
        elif op["op"] in FUSED:
            pending = (d, op)
        else:
            yield d, op, None
    assert pending is None, "a fused record without its partner"


def footprint_check(g, ops, precision, init, nphases=2):
    """the CPU walk over the records; returns the Footprints (its `valid` keys: every buffer a record touches)"""
    fp = Footprints(g, ESZ[precision])
    for (d, b), arr in init.items():
        assert arr.size <= fp.size(d)
        fp.region(d, b)[: arr.size] = 1
    for o in ops:
        for op in o:
            if "mult" in op:      # the convolution X pass also reads the multiplier through its load map
                for box in boxes(dict(op, **{"in": op["mult"]}), "i"):
                    mark(fp, box, "read", None)
    walk(fp, ops, nphases)
    return fp


class Replay:
    """the arenas of one replay.  init: {(device, buffer): flat array} (bufferDev1 inputs, multipliers, an in-place input)"""

    def __init__(self, g, ops, precision, init, nphases=2, mem=None, seed=7):
        self.g, self.ops, self.prec, self.nphases = g, ops, precision, nphases
        self.esz = ESZ[precision]
        self.fp = footprint_check(g, ops, precision, init, nphases)
        self.mem = mem or TorchMemory()
        npdt = NPDT[precision]
        rng = np.random.default_rng(seed)
        self.arena, self.base, self.pattern = {}, {}, {}
        for key in sorted(set(self.fp.valid) | set(init)):
            n = self.fp.size(key[0])
            host = np.full(CANARY + n + CANARY, complex(np.nan, np.nan), dtype=npdt)
            host[:CANARY] = rng.standard_normal(CANARY) + 1j * rng.standard_normal(CANARY)
            host[-CANARY:] = rng.standard_normal(CANARY) + 1j * rng.standard_normal(CANARY)
            if key in init:
                host[CANARY: CANARY + init[key].size] = init[key]
            self.pattern[key] = host
            self.arena[key], self.base[key] = self.mem.alloc(host)

    def ptr(self, addr):
        if not addr:
            return None
        d, b, off = self.fp.decode(addr)
        return self.base[(d, b)] + (CANARY + off) * self.esz

    def device_record(self, op):
        r = dict(op)
        for k in ("in", "out", "mult"):
            if k in r:
                r[k] = self.ptr(r[k])
        for side in ("ci", "co"):
            if side in r:
                r[side] = dict(r[side], cptr=[self.ptr(a) for a in r[side]["cptr"]])
        return r

    def run(self, launch=None):
        """launch every record once, in order; returns the number of launches (a fused pair counts once)"""
        launch = launch or dfft.debug_launch_op
        n = 0
        for d, op, second in launch_units(self.ops, self.nphases):
            if op["op"] == "alltoall":
                self.alltoall(d, op)
                continue
            rc = launch(self.device_record(op), self.prec, self.device_record(second) if second else None)
            assert rc == 0, (d, op["op"], rc, dfft.lib().dfft_last_error().decode())
            n += 1
        return n

    def alltoall(self, d, op):
        sd, sb, soff = self.fp.decode(op["send"])
        _, rb, roff = self.fp.decode(op["recv"])
        for q, so, ro, cnt in op["chunks"]:
            if cnt:
                dst = self.base[(q, rb)] + (CANARY + roff + ro) * self.esz
                src = self.base[(sd, sb)] + (CANARY + soff + so) * self.esz
                dfft.memcpy_dtod(dst, src, cnt * self.esz)

    def contents(self, outputs, keep=KEEP):
        """the arenas after the run; asserts every canary, that the buffers in `keep` are bitwise unchanged, and that
        outputs = {(device, buffer): count} hold no NaN in their first `count` elements.  Returns {key: those elements}"""
        got = {}
        for key, a in self.arena.items():
            host = self.mem.fetch(a)
            pat = self.pattern[key]
            bits = lambda x: np.ascontiguousarray(x).view(np.uint8)   # noqa: E731
            assert np.array_equal(bits(host[:CANARY]), bits(pat[:CANARY])), ("canary before", key)
            assert np.array_equal(bits(host[-CANARY:]), bits(pat[-CANARY:])), ("canary after", key)
            if key[1] in keep:
                assert np.array_equal(bits(host), bits(pat)), ("written", key)
            if key in outputs:
                v = host[CANARY: CANARY + outputs[key]]
                assert not np.isnan(v.view(v.real.dtype)).any(), ("NaN left in the output", key)
                got[key] = v.copy()
        return got


def slab_outputs(g, direction, inplace):
    """{(device, buffer): count} of the P output slabs of a C2C plan"""
    b = IN if inplace else 2
    return {(d, b): (g.out_count(d) if direction == dfft.FORWARD else g.in_count(d)) for d in range(g.P)}
