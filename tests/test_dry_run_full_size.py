"""CPU check of the multi-device schedules AT THE BASELINE'S FULL SIZES (512^3 .. 1024^3, 1..8 devices), without a GPU.

tests/test_dry_run.py gives the recorded passes of a DFFT_DRY_RUN plan their numerical meaning at sizes numpy can
transform in seconds.  What small sizes cannot show is the address arithmetic of the real configurations (BASELINE.json
configs 2-5): per-device counts of 2^27 elements, byte offsets beyond 2^32, part-major receive layouts with 4 z-parts,
8 senders.  Every pass is an affine map (a, b, c, e) -> address, optionally cut into per-peer chunks along e, so its read
and write footprints are unions of strided boxes: numpy strided views mark them on one byte per element, with no index
arrays.  Checked for every device, in program order (phase 0 of all devices, the all-to-alls, phase 1):
  * every address of every pass lies inside the buffer it names (of the device it names);
  * a pass never writes an element twice (the store map is injective);
  * a pass only reads elements that an earlier pass (or the caller's input) wrote -- in particular the X pass of a z-part
    reads exactly what the senders' Y passes of that part stored into this device's receive buffer;
  * at the end the output buffer holds exactly the device's output slab.
The kernels that execute these maps are checked against the oracle on the GPU (tests/test_gpu_*.py)."""
import numpy as np
import pytest
from numpy.lib.stride_tricks import as_strided

import distributedfft_b200 as dfft
from oracle import BACKWARD, FORWARD, SlabGeometry
from test_dry_run import schedule

BUF1, OUT, WORK, MID, IN = 1, 2, 3, 4, 5


def fake(dev, buf):
    return ((dev + 1) << 44) | (buf << 40)


class Footprints:
    def __init__(self, g, esz):
        self.g, self.esz = g, esz
        self.valid = {}          # (dev, buf) -> uint8[max_count]: 1 where some pass has stored (or the caller's input lies)
        self.counts = {}         # (dev, buf) -> uint8[max_count]: store counts of the pass being checked (reused, zeroed after use)

    def decode(self, addr):
        off = addr & ((1 << 40) - 1)
        assert off % self.esz == 0, "address not element-aligned"
        return (addr >> 44) - 1, (addr >> 40) & 0xF, off // self.esz

    def size(self, dev):
        return self.g.max_count(dev)

    def region(self, dev, buf):
        key = (dev, buf)
        if key not in self.valid:
            self.valid[key] = np.zeros(self.size(dev), dtype=np.uint8)
        return self.valid[key]


def boxes(op, side):
    """The strided boxes of a pass's load (side 'i') or store (side 'o') map: (base address, shape, strides in elements)."""
    N, C, G, W = op["N"], op["C"], op["G"], op["W"]
    A = op["ntiles"] // G
    assert A * G == op["ntiles"] and (G - 1) * C < W <= G * C
    SA, SB, cs, es = op["ia" if side == "i" else "oa"]
    ch = op.get("ci" if side == "i" else "co")
    runs = []          # (base, SA, e_count)
    if ch:
        for q in range(ch["nchunks"]):
            e0 = q * ch["ediv"]
            e1 = N if q == ch["nchunks"] - 1 else min(N, e0 + ch["ediv"])
            if e1 > e0:
                runs.append((ch["cptr"][q], ch["SAq"][q], e1 - e0))
    else:
        runs.append((op["in" if side == "i" else "out"], SA, N))
    out = []
    for base, sa, ne in runs:
        full_b, rag = W // C, W % C
        if full_b:
            out.append((base, (A, full_b, C, ne), (sa, SB, cs, es)))
        if rag:
            out.append((base + 0, (A, 1, rag, ne), (sa, SB, cs, es), full_b * SB))
    return out


def mark(fp, box, what, scratch):
    base, shape, strides = box[0], box[1], box[2]
    extra = box[3] if len(box) > 3 else 0
    dev, buf, off = fp.decode(base)
    off += extra
    assert 0 <= dev < fp.g.P, ("device", dev)
    assert all(s >= 0 for s in strides)
    last = off + sum((n - 1) * s for n, s in zip(shape, strides))
    assert off >= 0 and last < fp.size(dev), (what, "out of bounds", dev, buf, off, last, fp.size(dev))
    nel = int(np.prod(shape))
    if what == "read":
        v = as_strided(fp.region(dev, buf)[off:], shape=shape, strides=strides)
        assert v.all(), ("pass reads elements nobody wrote", dev, buf)
        return nel
    key = (dev, buf)
    if key not in fp.counts:
        fp.counts[key] = np.zeros(fp.size(dev), dtype=np.uint8)
    lo, hi = scratch.get(key, (off, last + 1))
    scratch[key] = (min(lo, off), max(hi, last + 1))          # the address range this pass touches in that buffer
    v = as_strided(fp.counts[key][off:], shape=shape, strides=strides)
    v += 1
    return nel


def run_pass(fp, op):
    nread = sum(mark(fp, b, "read", None) for b in boxes(op, "i"))
    scratch, nwritten = {}, 0
    for b in boxes(op, "o"):
        nwritten += mark(fp, b, "write", scratch)
    assert nread == nwritten == op["N"] * op["W"] * (op["ntiles"] // op["G"])
    total = 0
    for key, (lo, hi) in scratch.items():
        cnt = fp.counts[key][lo:hi]
        total += int(np.count_nonzero(cnt))       # nwritten increments landed on `total` distinct elements
        np.bitwise_or(fp.region(*key)[lo:hi], cnt, out=fp.region(*key)[lo:hi])
        cnt.fill(0)
    assert total == nwritten, ("store map writes an element twice", total, nwritten)


def run_alltoall(fp, dev, op):
    sdev, sbuf, soff = fp.decode(op["send"])
    rdev, rbuf, roff = fp.decode(op["recv"])
    assert sdev == dev == rdev
    for q, so, ro, cnt in op["chunks"]:
        assert 0 <= soff + so and soff + so + cnt <= fp.size(dev) and 0 <= roff + ro and roff + ro + cnt <= fp.size(q)
        assert fp.region(dev, sbuf)[soff + so: soff + so + cnt].all(), "all-to-all sends elements nobody wrote"
        fp.region(q, rbuf)[roff + ro: roff + ro + cnt] = 1


def walk(fp, ops, nphases=2):
    """every record of every device in the interpreters' order (test_dry_run.schedule) through the checks above"""
    for d, op in schedule(ops, nphases):
        if op["op"] == "alltoall":
            run_alltoall(fp, d, op)
        else:
            run_pass(fp, op)


def check(n0, n1, n2, P, direction, flags, precision=dfft.DOUBLE, mutate=None):
    need = 10 * n0 * n1 * n2            # one byte per element for ~4 buffers x (written + per-pass counts), all devices
    if need > 2 ** 30:
        import psutil
        if psutil.virtual_memory().available < 2 * need:
            pytest.skip(f"needs ~{need >> 30} GiB of host memory for the footprint maps")
    g = SlabGeometry(n0, n1, n2, P)
    fp = Footprints(g, 16 if precision == dfft.DOUBLE else 8)
    plans, ops = [], []
    for d in range(P):
        cnt_in = g.in_count(d) if direction == FORWARD else g.out_count(d)
        fp.region(d, BUF1)[:cnt_in] = 1                # the plan snapshots `in` into bufferDev1 (api.cpp:76-77)
        plans.append(dfft.fft_mpi_plan_dft_c2c_3d(n0, n1, n2, fake(d, IN), fake(d, OUT), None, d, P, direction, precision, flags | dfft.DRY_RUN))
    for p in plans:
        p.execute()
        ops.append(p.recorded_ops())
    if mutate:
        mutate(ops)
    walk(fp, ops)
    for d in range(P):
        cnt_out = g.out_count(d) if direction == FORWARD else g.in_count(d)
        out = fp.region(d, OUT)
        assert out[:cnt_out].all(), ("output slab not covered", d)
        if g.n0 % P == 0 and g.n1 % P == 0:      # (with a short last slab `out` is max_count long and doubles as a work buffer)
            assert not out[cnt_out:].any(), ("stores beyond the output slab", d)
    info = dict(names=[[op["op"] for op in o] for o in ops], parts=plans[0].pipeline_parts, chain=plans[0].pipeline_chain, fused=plans[0].fused)
    for p in plans:
        p.destroy()
    return info


P2P, NCCL, PIPE, NOPIPE = dfft.EXCHANGE_P2P, dfft.EXCHANGE_NCCL, dfft.FORCE_PIPELINE, dfft.NO_PIPELINE

# BASELINE.json configs 2-5 (+ the 2- and 8-device variants of config 3 the scaling run uses), default flags
BASELINE_CASES = [("C2 512^3 P1", 512, 1, dfft.DOUBLE), ("C3c 512^3 P2", 512, 2, dfft.DOUBLE), ("C3 512^3 P4", 512, 4, dfft.DOUBLE), ("C3b 512^3 P8", 512, 8, dfft.DOUBLE),
                  ("C4 1024^3 P8", 1024, 8, dfft.DOUBLE), ("C5 768^3 fp32 P8", 768, 8, dfft.FLOAT)]


@pytest.mark.parametrize("name,n,P,precision", BASELINE_CASES, ids=[c[0] for c in BASELINE_CASES])
def test_baseline_configs_default_schedule_footprints(name, n, P, precision):
    for direction in (FORWARD, BACKWARD):
        info = check(n, n, n, P, direction, P2P if P > 1 else 0, precision)
        if direction == FORWARD and P >= 4 and n >= 1024:
            # the default there is the kernel chain [Z + Y0] [Y1 + X0] ... [X last] over 4 z-parts (DESIGN.md 5.1)
            assert info["chain"] and info["parts"] == 4 and info["names"][0] == ["fusedZ", "fusedY"] + ["Y_CO", "XF"] * 3 + ["XF"]
        else:
            assert info["parts"] == 0


@pytest.mark.parametrize("n,P,flags,direction", [
    (512, 4, P2P | PIPE, FORWARD), (512, 8, P2P | PIPE, FORWARD), (512, 8, P2P | PIPE, BACKWARD), (512, 2, P2P | PIPE, FORWARD),
    (512, 8, NCCL | PIPE, FORWARD), (512, 8, NCCL | PIPE, BACKWARD), (512, 4, NCCL, FORWARD), (512, 8, NCCL | NOPIPE, BACKWARD),
    (512, 8, P2P | dfft.NO_FUSE, FORWARD), (1024, 8, P2P | NOPIPE, FORWARD),
    (1024, 8, NCCL | PIPE, FORWARD)])
def test_every_multi_device_schedule_at_full_size(n, P, flags, direction):
    info = check(n, n, n, P, direction, flags)
    if flags & PIPE:
        assert info["parts"] in (2, 4)
    if flags & NOPIPE:
        assert info["parts"] == 0


def test_two_stream_pipeline_and_uneven_full_size(monkeypatch):
    monkeypatch.setenv("DFFT_PIPE_MODE", "streams")
    info = check(512, 512, 512, 4, FORWARD, P2P | PIPE)
    assert info["parts"] == 4 and not info["chain"]
    monkeypatch.delenv("DFFT_PIPE_MODE")
    # uneven splits at a realistic size (short last slab in x and in y): 500 x 300 x 512 over 8 and over 3 devices
    for P in (8, 3):
        for direction in (FORWARD, BACKWARD):
            check(500, 300, 512, P, direction, P2P)
            check(500, 300, 512, P, direction, NCCL)


def test_the_checker_itself_catches_broken_maps():
    """Mutation test of this file's checker on a small chain schedule: each kind of damage to a recorded map must trip it."""
    args = (64, 64, 64, 4, FORWARD, P2P | PIPE)
    assert check(*args)["chain"]

    def first(ops, name, dev=1):
        return next(op for op in ops[dev] if op["op"] == name)

    def beyond_the_buffer(ops):
        for op in ops[1]:
            if op["op"] == "XF":
                op["out"] += 16 * 64                  # the X stores slide 64 elements: the last plane's fall off the end
    def double_store(ops):
        first(ops, "Y_CO")["oa"][1] = 0               # every column group of a Y part lands on the same rows
    def lost_sender(ops):
        last = [op for op in ops[2] if op["op"] == "Y_CO"][-1]
        ops[2][:] = [op for op in ops[2] if op is not last]              # device 2 never sends its last z-part
    def shifted_peer_base(ops):
        first(ops, "fusedY")["co"]["cptr"][0] += 16 * 16                # device 1's block in device 0's receive buffer starts a row late
    # (what footprints cannot see -- the right elements in the wrong order or at the wrong peer -- is what test_dry_run.py's
    # numerical interpreter is for)
    for damage in (beyond_the_buffer, double_store, lost_sender, shifted_peer_base):
        with pytest.raises(AssertionError):
            check(*args, mutate=damage)
