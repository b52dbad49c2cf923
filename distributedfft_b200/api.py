"""ctypes binding of libdfft.so mirroring the reference's slab-FFT API.

Reference surface (3dmpifft_opt/include/fft_mpi_3d_api.h:68-74, fft_mpi_common.h:15-22):
    fft_mpi_init, fft_mpi_plan_dft_c2c_3d, fft_mpi_execute_dft_3d_c2c, fft_mpi_destroy_plan,
    fft_mpi_alloc_local_memory, fft_mpi_local_size_3d, fft_mpi_cleanup, getMaxDataCount,
    FORWARD / BACKWARD, ALLOC_CPU / ALLOC_DEV.
Same names, argument meaning and error behaviour (errors raise DfftError instead of exit()).
Device memory is handled as raw pointers; callers may pass torch CUDA tensors' data_ptr().
"""
from __future__ import annotations

import ctypes
import os

FORWARD = 1
BACKWARD = -1
ALLOC_CPU = 1
ALLOC_DEV = -1
DOUBLE = 0
FLOAT = 1
EXCHANGE_AUTO, EXCHANGE_P2P, EXCHANGE_NCCL, EXCHANGE_STAGED = 0, 1, 2, 3
SCALE_BACKWARD = 4
NO_FUSE = 8
FORCE_FUSE = 16
OVERLAP_X = 32
NATURAL_SPECTRUM = 64
DRY_RUN = 128
NO_PIPELINE = 256
NO_TMA = 512
FORCE_PIPELINE = 1024

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdfft.so")

__all__ = [
    "FORWARD", "BACKWARD", "ALLOC_CPU", "ALLOC_DEV", "DOUBLE", "FLOAT", "EXCHANGE_AUTO", "EXCHANGE_P2P",
    "EXCHANGE_NCCL", "EXCHANGE_STAGED", "SCALE_BACKWARD", "NO_FUSE", "FORCE_FUSE", "OVERLAP_X", "NATURAL_SPECTRUM", "DRY_RUN", "NO_PIPELINE", "NO_TMA", "FORCE_PIPELINE", "DfftError", "lib", "LIB_PATH", "Plan", "LocalComm",
    "BootstrapComm", "fft_mpi_init", "fft_mpi_plan_dft_c2c_3d", "fft_mpi_execute_dft_3d_c2c", "fft_mpi_destroy_plan",
    "fft_mpi_alloc_local_memory", "fft_mpi_local_size_3d", "fft_mpi_cleanup", "getMaxDataCount", "supported_lengths",
    "fft_mpi_plan_dft_r2c_3d", "local_size_r2c_3d", "fft_mpi_plan_dft_convolve_3d",
    "fft_lines", "lines_ops", "LinesPlan", "RealLinesPlan", "real_lines_ops", "lines_3d_ops", "LinesConvolvePlan", "lines_conv_3d_ops", "lines_conv_2d_ops", "lines_conv_1d_ops", "lines_conv_padded_1d_ops", "length_kind", "length_schedule", "memcpy_htod", "memcpy_dtoh", "memcpy_dtod", "debug_launch_op", "exchange_table", "comm_allgather",
]


class DfftError(RuntimeError):
    pass


_ALLGATHER = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)
_lib = None


class _DebugChunks(ctypes.Structure):
    _fields_ = [("ediv", ctypes.c_int), ("nchunks", ctypes.c_int), ("cptr", ctypes.c_void_p * 32), ("SAq", ctypes.c_longlong * 32)]


class _DebugOp(ctypes.Structure):
    """dfft_debug_op (dfft.h)"""
    _fields_ = [("N", ctypes.c_int), ("C", ctypes.c_int), ("G", ctypes.c_int), ("W", ctypes.c_int), ("ntiles", ctypes.c_longlong),
                ("inv", ctypes.c_int), ("do_scale", ctypes.c_int), ("scale", ctypes.c_double), ("tw_n", ctypes.c_longlong),
                ("in_", ctypes.c_void_p), ("out", ctypes.c_void_p), ("mult", ctypes.c_void_p),
                ("ia", ctypes.c_longlong * 4), ("oa", ctypes.c_longlong * 4), ("ci", _DebugChunks), ("co", _DebugChunks)]


def lib():
    """Load libdfft.so; raises (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DfftError(f"{LIB_PATH} is missing: build it with `python -m distributedfft_b200.build` "
                        "(there is no CPU fallback)")
    L = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    ll, i, vp, u = ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint
    P = ctypes.POINTER
    L.dfft_last_error.restype = ctypes.c_char_p
    L.dfft_version.restype = i
    L.dfft_supported_lengths.argtypes = [i, P(i), i]
    L.dfft_init.argtypes = [P(ll), i, P(i), P(i), P(ll)]
    L.dfft_max_data_count.argtypes = [ll, ll, ll, i, i]
    L.dfft_max_data_count.restype = ll
    L.dfft_local_size_3d.argtypes = [ll, ll, ll, i, i, P(ll), P(ll), P(ll), P(ll)]
    L.dfft_local_size_3d.restype = ll
    L.dfft_alloc_local.argtypes = [ll, i, i]
    L.dfft_alloc_local.restype = vp
    L.dfft_free_local.argtypes = [vp, i]
    L.dfft_comm_create_local.argtypes = [i, P(vp)]
    L.dfft_comm_create_bootstrap.argtypes = [i, i, _ALLGATHER, vp, P(vp)]
    L.dfft_comm_destroy.argtypes = [vp]
    L.dfft_comm_allgather.argtypes = [vp, i, vp, vp, ctypes.c_size_t]
    L.dfft_exchange_table.argtypes = [ll, ll, ll, i, i, i, P(ll), P(ll), P(ll), P(ll)]
    L.dfft_plan_c2c_3d.argtypes = [ll, ll, ll, vp, vp, vp, i, i, i, i, u, P(vp)]
    L.dfft_plan_r2c_3d.argtypes = [ll, ll, ll, vp, vp, vp, i, i, i, i, u, P(vp)]
    L.dfft_local_size_r2c_3d.argtypes = [ll, ll, ll, i, i, P(ll), P(ll)]
    L.dfft_plan_convolve_c2c_3d.argtypes = [ll, ll, ll, vp, vp, vp, i, i, i, u, P(vp)]
    L.dfft_plan_convolve_r2c_3d.argtypes = [ll, ll, ll, vp, vp, vp, i, i, i, u, P(vp)]
    L.dfft_execute_convolve.argtypes = [vp, vp]
    for name in ("dfft_execute", "dfft_synchronize", "dfft_destroy", "dfft_plan_launches", "dfft_plan_exchange", "dfft_plan_fused", "dfft_plan_pipeline_parts", "dfft_plan_tma_mask", "dfft_plan_pipeline_chain"):
        getattr(L, name).argtypes = [vp]
    L.dfft_execute_stage.argtypes = [vp, i]
    L.dfft_execute_host.argtypes = [vp, vp, vp]
    L.dfft_execute_host_async.argtypes = [vp, vp, vp]
    L.dfft_get_timings.argtypes = [vp, P(ctypes.c_double)]
    L.dfft_get_pass_timings.argtypes = [vp, P(ctypes.c_double)]
    L.dfft_plan_buffers.argtypes = [vp, P(vp), P(vp)]
    L.dfft_plan_counts.argtypes = [vp, P(ll), P(ll), P(ll)]
    L.dfft_plan_stream.argtypes = [vp]
    L.dfft_plan_stream.restype = vp
    L.dfft_fft_lines.argtypes = [vp, i, ll, ll, ll, ll, ll, i, i]
    L.dfft_lines_plan_create.argtypes = [i, ll, ll, ll, ll, ll, i, P(vp)]
    L.dfft_lines_plan_create_2d.argtypes = [i, i, ll, i, P(vp)]
    L.dfft_lines_execute.argtypes = [vp, vp, i]
    L.dfft_lines_synchronize.argtypes = [vp]
    L.dfft_lines_destroy.argtypes = [vp]
    L.dfft_lines_stream.argtypes = [vp]
    L.dfft_lines_stream.restype = vp
    L.dfft_lines_plan_create_r2c.argtypes = [i, ll, i, P(vp)]
    L.dfft_lines_plan_create_r2c_2d.argtypes = [i, i, ll, i, P(vp)]
    L.dfft_lines_execute_real.argtypes = [vp, vp, vp, i]
    L.dfft_lines_plan_create_3d.argtypes = [i, i, i, ll, i, P(vp)]
    L.dfft_lines_plan_create_r2c_3d.argtypes = [i, i, i, ll, i, P(vp)]
    L.dfft_debug_lines_3d_ops.argtypes = [i, i, i, ll, i, i, i, ctypes.c_char_p, ll]
    L.dfft_debug_lines_3d_ops.restype = ll
    L.dfft_lines_plan_create_convolve_3d.argtypes = [i, i, i, ll, i, ctypes.c_uint, P(vp)]
    L.dfft_lines_plan_create_convolve_r2c_3d.argtypes = [i, i, i, ll, i, ctypes.c_uint, P(vp)]
    L.dfft_lines_execute_convolve.argtypes = [vp, vp, vp, vp, ll]
    L.dfft_debug_lines_conv_3d_ops.argtypes = [i, i, i, ll, i, i, ctypes.c_uint, ll, ctypes.c_char_p, ll]
    L.dfft_debug_lines_conv_3d_ops.restype = ll
    L.dfft_lines_plan_create_convolve_2d.argtypes = [i, i, ll, i, ctypes.c_uint, P(vp)]
    L.dfft_lines_plan_create_convolve_r2c_2d.argtypes = [i, i, ll, i, ctypes.c_uint, P(vp)]
    L.dfft_debug_lines_conv_2d_ops.argtypes = [i, i, ll, i, i, ctypes.c_uint, ll, ctypes.c_char_p, ll]
    L.dfft_debug_lines_conv_2d_ops.restype = ll
    L.dfft_lines_plan_create_convolve_1d.argtypes = [i, ll, i, ctypes.c_uint, P(vp)]
    L.dfft_lines_plan_create_convolve_r2c_1d.argtypes = [i, ll, i, ctypes.c_uint, P(vp)]
    L.dfft_debug_lines_conv_1d_ops.argtypes = [i, ll, i, i, ctypes.c_uint, ll, ctypes.c_char_p, ll]
    L.dfft_debug_lines_conv_1d_ops.restype = ll
    L.dfft_lines_plan_create_convolve_padded_1d.argtypes = [i, ll, ll, ll, i, ctypes.c_uint, P(vp)]
    L.dfft_debug_lines_conv_padded_1d_ops.argtypes = [i, ll, ll, ll, i, ctypes.c_uint, ll, ctypes.c_char_p, ll]
    L.dfft_debug_lines_conv_padded_1d_ops.restype = ll
    L.dfft_lines_plan_create_convolve_padded_r2c_1d.argtypes = [i, ll, ll, ll, i, ctypes.c_uint, P(vp)]
    L.dfft_debug_lines_conv_padded_r2c_1d_ops.argtypes = [i, ll, ll, ll, i, ctypes.c_uint, ll, ctypes.c_char_p, ll]
    L.dfft_debug_lines_conv_padded_r2c_1d_ops.restype = ll
    L.dfft_debug_real_lines_ops.argtypes = [i, i, ll, i, i, i, ctypes.c_char_p, ll]
    L.dfft_debug_real_lines_ops.restype = ll
    L.dfft_length_kind.argtypes = [i, i]
    L.dfft_debug_plan_ops.argtypes = [vp, ctypes.c_char_p, ll]
    L.dfft_debug_plan_ops.restype = ll
    L.dfft_debug_launch_op.argtypes = [ctypes.c_char_p, P(_DebugOp), ctypes.c_char_p, P(_DebugOp), i]
    L.dfft_debug_lines_ops.argtypes = [i, ll, ll, ll, ll, ll, i, i, i, ctypes.c_char_p, ll]
    L.dfft_debug_lines_ops.restype = ll
    L.dfft_length_schedule.argtypes = [i, i, P(ctypes.c_int), i]
    L.dfft_debug_fused3_order.argtypes = [ll, ll, i, i, i, i, i, ll, P(ll)]
    L.dfft_debug_fused3_order.restype = ll
    L.dfft_debug_fused2_order.argtypes = [ll, i, i, i, ll, P(ll)]
    L.dfft_debug_fused2_order.restype = ll
    L.dfft_memcpy.argtypes = [vp, vp, ctypes.c_size_t, i]
    L.dfft_debug_timeline.argtypes = [vp, P(ctypes.c_double)]
    _lib = L
    return L


def _check(rc, what):
    if rc != 0:
        raise DfftError(f"{what} failed ({rc}): {lib().dfft_last_error().decode()}")


def supported_lengths(precision=DOUBLE):
    n = lib().dfft_supported_lengths(precision, None, 0)
    arr = (ctypes.c_int * n)()
    lib().dfft_supported_lengths(precision, arr, n)
    return list(arr)


def length_kind(n, precision=DOUBLE):
    """2 = tuned kernel, 1 = run-time-scheduled kernel (2..13-smooth lengths), 0 = unsupported."""
    return int(lib().dfft_length_kind(n, precision))


def length_schedule(n, precision=DOUBLE):
    """radix list the library uses for length n ([] if unsupported)"""
    arr = (ctypes.c_int * 32)()
    k = lib().dfft_length_schedule(n, precision, arr, 32)
    return list(arr[:k])


def getMaxDataCount(n0, n1, n2, totalDevCount, isLastDevice):
    """getMaxDataCount, fft_mpi_3d_api.cpp:289-316"""
    return int(lib().dfft_max_data_count(n0, n1, n2, totalDevCount, int(bool(isLastDevice))))


def fft_mpi_init(N, iniDeviceNumInNode):
    """fft_mpi_init (fft_mpi_3d_api.cpp:3-39). Returns (newDeviceCount, newDeviceCountInNode, dataCountInNode)."""
    n = (ctypes.c_longlong * 3)(*N)
    tot, loc = ctypes.c_int(0), ctypes.c_int(0)
    counts = (ctypes.c_longlong * max(1, iniDeviceNumInNode))()
    _check(lib().dfft_init(n, iniDeviceNumInNode, ctypes.byref(tot), ctypes.byref(loc), counts), "fft_mpi_init")
    return tot.value, loc.value, list(counts[: tot.value])


def fft_mpi_local_size_3d(n0, n1, n2, totalDevCount, devIdx):
    """declared fft_mpi_3d_api.h:73; returns (alloc, local_n0, local_0_start, local_n1, local_1_start)"""
    a, b, c, d = (ctypes.c_longlong(0) for _ in range(4))
    r = lib().dfft_local_size_3d(n0, n1, n2, totalDevCount, devIdx, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c), ctypes.byref(d))
    if r < 0:
        raise DfftError("fft_mpi_local_size_3d: bad arguments")
    return int(r), a.value, b.value, c.value, d.value


def fft_mpi_alloc_local_memory(count, flag, precision=DOUBLE):
    """fft_mpi_alloc_local_memory (fft_mpi_3d_api.cpp:216-230); returns a raw pointer (int)."""
    p = lib().dfft_alloc_local(count, flag, precision)
    if not p:
        raise DfftError("fft_mpi_alloc_local_memory: " + lib().dfft_last_error().decode())
    return p


def exchange_table(n0, n1, n2, totalDevCount, devIdx, direction):
    """TransInfo of one device (fft_mpi_3d_api.cpp:84-133): dict of scount/soffset/rcount/roffset lists."""
    arrs = [(ctypes.c_longlong * totalDevCount)() for _ in range(4)]
    _check(lib().dfft_exchange_table(n0, n1, n2, totalDevCount, devIdx, direction, *arrs), "dfft_exchange_table")
    return dict(zip(("scount", "soffset", "rcount", "roffset"), (list(x) for x in arrs)))


def comm_allgather(comm, rank, payload: bytes):
    """All-gather `payload` through a dfft communicator (the plan-creation bootstrap path)."""
    n = comm.nranks
    buf = ctypes.create_string_buffer(len(payload) * n)
    _check(lib().dfft_comm_allgather(comm.handle, rank, payload, buf, len(payload)), "dfft_comm_allgather")
    return [buf.raw[i * len(payload):(i + 1) * len(payload)] for i in range(n)]


def fft_mpi_cleanup():
    lib().dfft_cleanup()


class LocalComm:
    """P device-threads of one process (the reference's GPUs-per-rank mode)."""

    def __init__(self, nranks):
        h = ctypes.c_void_p()
        _check(lib().dfft_comm_create_local(nranks, ctypes.byref(h)), "dfft_comm_create_local")
        self.handle, self.nranks = h, nranks

    def destroy(self):
        if self.handle:
            lib().dfft_comm_destroy(self.handle)
            self.handle = None


class BootstrapComm:
    """One process per GPU; `allgather(bytes) -> list[bytes]` supplied by the host program
    (e.g. torch.distributed.all_gather_object).  Stands in for the reference's MPI_Comm."""

    def __init__(self, rank, nranks, allgather):
        self._py_allgather = allgather

        def _cb(ctx, send, recv, nbytes):
            try:
                mine = ctypes.string_at(send, nbytes)
                parts = self._py_allgather(mine)
                assert len(parts) == nranks and all(len(x) == nbytes for x in parts)
                ctypes.memmove(recv, b"".join(parts), nbytes * nranks)
                return 0
            except Exception as exc:  # pragma: no cover - surfaced as DFFT_ECOMM
                print("dfft bootstrap allgather failed:", exc)
                return -1

        self._cb = _ALLGATHER(_cb)
        h = ctypes.c_void_p()
        _check(lib().dfft_comm_create_bootstrap(rank, nranks, self._cb, None, ctypes.byref(h)), "dfft_comm_create_bootstrap")
        self.handle, self.nranks, self.rank = h, nranks, rank

    def destroy(self):
        if self.handle:
            lib().dfft_comm_destroy(self.handle)
            self.handle = None


class Plan:
    """fft_mpi_3d_plan (fft_mpi_3d_api.h:11-66): bufferDev1/bufferDev2, counts, timings."""

    def __init__(self, handle):
        self.handle = handle
        b1, b2 = ctypes.c_void_p(), ctypes.c_void_p()
        _check(lib().dfft_plan_buffers(handle, ctypes.byref(b1), ctypes.byref(b2)), "dfft_plan_buffers")
        self.bufferDev1, self.bufferDev2 = b1.value, b2.value
        a, b, c = (ctypes.c_longlong(0) for _ in range(3))
        _check(lib().dfft_plan_counts(handle, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)), "dfft_plan_counts")
        self.in_count, self.out_count, self.maxDataCountInDevice = a.value, b.value, c.value

    def execute(self):
        _check(lib().dfft_execute(self.handle), "fft_mpi_execute_dft_3d_c2c")

    def execute_convolve(self, mult_ptr):
        """convolve plans: out = inverse(m .* forward(bufferDev1)) with the multiplier at `mult_ptr` (see
        fft_mpi_plan_dft_convolve_3d)"""
        _check(lib().dfft_execute_convolve(self.handle, mult_ptr), "dfft_execute_convolve")

    def execute_stage(self, stage):
        _check(lib().dfft_execute_stage(self.handle, stage), "dfft_execute_stage")

    def execute_host(self, host_in_ptr, host_out_ptr):
        _check(lib().dfft_execute_host(self.handle, host_in_ptr, host_out_ptr), "dfft_execute_host")

    def execute_host_async(self, host_in_ptr, host_out_ptr):
        _check(lib().dfft_execute_host_async(self.handle, host_in_ptr, host_out_ptr), "dfft_execute_host_async")

    def synchronize(self):
        _check(lib().dfft_synchronize(self.handle), "dfft_synchronize")

    def timings(self):
        t = (ctypes.c_double * 5)()
        _check(lib().dfft_get_timings(self.handle, t), "dfft_get_timings")
        return list(t)

    def pass_timings(self):
        t = (ctypes.c_double * 3)()
        _check(lib().dfft_get_pass_timings(self.handle, t), "dfft_get_pass_timings")
        return list(t)

    @property
    def launches(self):
        return lib().dfft_plan_launches(self.handle)

    @property
    def exchange(self):
        return lib().dfft_plan_exchange(self.handle)

    @property
    def fused(self):
        return bool(lib().dfft_plan_fused(self.handle))

    def recorded_ops(self):
        """passes recorded by the last execute of a DRY_RUN plan (list of dicts)"""
        import json
        n = lib().dfft_debug_plan_ops(self.handle, None, 0)
        buf = ctypes.create_string_buffer(int(n))
        lib().dfft_debug_plan_ops(self.handle, buf, n)
        return json.loads(buf.value.decode())

    def debug_timeline(self):
        t = (ctypes.c_double * 11)()
        _check(lib().dfft_debug_timeline(self.handle, t), "dfft_debug_timeline")
        return list(t)

    @property
    def tma_mask(self):
        """bit 0 / 1 / 2: the un-chunked Z / Y / X pass runs on the TMA-pipelined kernel"""
        return lib().dfft_plan_tma_mask(self.handle)

    @property
    def pipeline_parts(self):
        """z-parts of the stream-pipelined forward path (0 = not pipelined)"""
        return lib().dfft_plan_pipeline_parts(self.handle)

    @property
    def pipeline_chain(self):
        """the z-parts run as a chain of two-role kernels on one stream (Y part k + X part k-1 per kernel)"""
        return bool(lib().dfft_plan_pipeline_chain(self.handle))

    @property
    def overlapped(self):
        """forward transform runs as the single overlapped kernel (OVERLAP_X, experimental)"""
        return lib().dfft_plan_fused(self.handle) == 2

    @property
    def stream(self):
        return lib().dfft_plan_stream(self.handle)

    def destroy(self):
        if self.handle:
            lib().dfft_destroy(self.handle)
            self.handle = None


def fft_mpi_plan_dft_c2c_3d(n0, n1, n2, in_ptr, out_ptr, comm, devIdx, totalDevCount, direction, precision=DOUBLE, flags=0):
    """fft_mpi_plan_dft_c2c_3d (fft_mpi_3d_api.cpp:41-141). `comm` is a LocalComm/BootstrapComm (None for 1 device);
    the `node_data` array of the reference is owned by the communicator here."""
    h = ctypes.c_void_p()
    ch = comm.handle if comm is not None else None
    _check(lib().dfft_plan_c2c_3d(n0, n1, n2, in_ptr, out_ptr, ch, devIdx, totalDevCount, direction, precision, flags, ctypes.byref(h)),
           "fft_mpi_plan_dft_c2c_3d")
    return Plan(h)


def fft_mpi_plan_dft_r2c_3d(n0, n1, n2, in_ptr, out_ptr, comm, devIdx, totalDevCount, direction, precision=DOUBLE, flags=0):
    """Real-to-complex (FORWARD) / complex-to-real (BACKWARD) slab transform (dfft_plan_r2c_3d).  FORWARD: `in_ptr` holds the
    real x-slab [x_l][y][z], `out_ptr` receives the half spectrum [y_l][n2//2+1][x]; BACKWARD is the exact inverse layout,
    unnormalised unless SCALE_BACKWARD.  Buffer sizes: local_size_r2c_3d; `out_ptr` must be a separate buffer.  Plan.in_count /
    out_count are in elements of their own type (reals or complex)."""
    h = ctypes.c_void_p()
    ch = comm.handle if comm is not None else None
    _check(lib().dfft_plan_r2c_3d(n0, n1, n2, in_ptr, out_ptr, ch, devIdx, totalDevCount, direction, precision, flags, ctypes.byref(h)),
           "fft_mpi_plan_dft_r2c_3d")
    return Plan(h)


def fft_mpi_plan_dft_convolve_3d(n0, n1, n2, in_ptr, out_ptr, comm, devIdx, totalDevCount, precision=DOUBLE, flags=0, real=False):
    """Spectral convolution plan (dfft_plan_convolve_c2c_3d / dfft_plan_convolve_r2c_3d): Plan.execute_convolve(mult_ptr) computes
    out = ifftn(fftn(in) * m), unnormalised (x n0*n1*n2) unless SCALE_BACKWARD, or with real=True
    out = irfftn(rfftn(in) * m, s=(n0, n1, n2)) * n0*n1*n2 on real slabs.  `in_ptr` / `out_ptr` hold exactly this device's x-slab
    [x_l][y][z] (out_ptr None or == in_ptr: in place).  The complex multiplier is m[x][y_l][z'] in natural order over this
    device's y-slab (fft_mpi_local_size_3d), z' < n2, or n2//2+1 with real=True."""
    h = ctypes.c_void_p()
    ch = comm.handle if comm is not None else None
    fn = lib().dfft_plan_convolve_r2c_3d if real else lib().dfft_plan_convolve_c2c_3d
    _check(fn(n0, n1, n2, in_ptr, out_ptr, ch, devIdx, totalDevCount, precision, flags, ctypes.byref(h)), "fft_mpi_plan_dft_convolve_3d")
    return Plan(h)


def local_size_r2c_3d(n0, n1, n2, totalDevCount, devIdx):
    """(real_count, complex_count) of one device: reals of its x-slab, complex elements of its half-spectrum y-slab"""
    r, c = ctypes.c_longlong(0), ctypes.c_longlong(0)
    _check(lib().dfft_local_size_r2c_3d(n0, n1, n2, totalDevCount, devIdx, ctypes.byref(r), ctypes.byref(c)), "dfft_local_size_r2c_3d")
    return r.value, c.value


def fft_mpi_execute_dft_3d_c2c(plan: Plan):
    plan.execute()


def fft_mpi_destroy_plan(plan: Plan):
    plan.destroy()


def memcpy_htod(dev_ptr, host_ptr, nbytes):
    _check(lib().dfft_memcpy(dev_ptr, host_ptr, nbytes, 1), "dfft_memcpy")


def memcpy_dtoh(host_ptr, dev_ptr, nbytes):
    _check(lib().dfft_memcpy(host_ptr, dev_ptr, nbytes, 2), "dfft_memcpy")


def memcpy_dtod(dst_ptr, src_ptr, nbytes):
    _check(lib().dfft_memcpy(dst_ptr, src_ptr, nbytes, 0), "dfft_memcpy")


class _LinesPlanBase:
    """what the three lines plan classes share: the plan handle, its stream, synchronize and destroy"""

    def _create(self, name, *args):
        h = ctypes.c_void_p()
        _check(getattr(lib(), name)(*args, ctypes.byref(h)), name)
        self.handle = h

    def synchronize(self):
        _check(lib().dfft_lines_synchronize(self.handle), "dfft_lines_synchronize")

    @property
    def stream(self):
        return lib().dfft_lines_stream(self.handle)

    def destroy(self):
        if self.handle:
            lib().dfft_lines_destroy(self.handle)
            self.handle = None


class LinesPlan(_LinesPlanBase):
    """templateFFT engine surface (templateFFT.h:361-365): initializeFFT -> LinesPlan(...), launchFFTKernel -> execute,
    deleteFFT -> destroy.  Batched 1-D lines (contiguous or strided), with `two_d=(nx, ny, batch)` batched 2-D, or with
    `three_d=(nx, ny, nz, batch)` batched 3-D (numpy.fft.fftn over the last three axes of a[batch][nz][ny][nx])."""

    def __init__(self, n=None, stride=1, nlines=0, inner=0, inner_dist=0, outer_dist=0, precision=DOUBLE, two_d=None, three_d=None):
        if three_d is not None:
            self._create("dfft_lines_plan_create_3d", *three_d, precision)
        elif two_d is not None:
            self._create("dfft_lines_plan_create_2d", two_d[0], two_d[1], two_d[2], precision)
        else:
            self._create("dfft_lines_plan_create", n, stride, nlines, inner, inner_dist, outer_dist, precision)

    def execute(self, ptr, direction):
        _check(lib().dfft_lines_execute(self.handle, ptr, direction), "dfft_lines_execute")


class RealLinesPlan(_LinesPlanBase):
    """Real-data lines: R2C (FORWARD) / C2R (BACKWARD, unnormalised), out of place.  `nlines` densely packed real lines of `n`
    points <-> as many half spectra of n//2+1 complex points, or, with `two_d=(nx, ny, batch)`, `batch` row-major ny x nx real
    matrices <-> ny x (nx//2+1) complex matrices (numpy.fft.rfft2 layout), or, with `three_d=(nx, ny, nz, batch)`, nz x ny x nx
    real arrays <-> nz x ny x (nx//2+1) complex arrays (numpy.fft.rfftn layout)."""

    def __init__(self, n=None, nlines=0, precision=DOUBLE, two_d=None, three_d=None):
        if three_d is not None:
            self._create("dfft_lines_plan_create_r2c_3d", *three_d, precision)
        elif two_d is not None:
            self._create("dfft_lines_plan_create_r2c_2d", two_d[0], two_d[1], two_d[2], precision)
        else:
            self._create("dfft_lines_plan_create_r2c", n, nlines, precision)

    def execute(self, in_ptr, out_ptr, direction):
        _check(lib().dfft_lines_execute_real(self.handle, in_ptr, out_ptr, direction), "dfft_lines_execute_real")


class LinesConvolvePlan(_LinesPlanBase):
    """Batched 3-D spectral convolution, `three_d=(nx, ny, nz, batch)`: out = ifftn(fftn(in) * m) over the last three axes of
    a[batch][nz][ny][nx], unnormalised (x nx*ny*nz) unless flags=SCALE_BACKWARD; with real=True, real in / real out,
    out = irfftn(rfftn(in) * m, s=(nz, ny, nx)) * nx*ny*nz.  m is complex in the plan's precision, [nz][ny][nx] (real:
    [nz][ny][nx//2+1]) per volume; execute with mult_count=1 shares one multiplier among all volumes, mult_count=batch gives
    each its own.  in_ptr == out_ptr runs in place; `in` and the multiplier are never written otherwise.
    `two_d=(nx, ny, batch)` instead: the same over the last two axes of a[batch][ny][nx] (m: [ny][nx], real: [ny][nx//2+1]
    per image).  `one_d=(n, nlines)` instead: out = ifft(fft(in) * m) per line of a[nlines][n] (m: [n], real: [n//2+1] per line),
    one kernel launch per execute.  Exactly one of one_d, two_d and three_d is given.
    `padded=(in_len, out_len)` with one_d (complex only): the zero-padded convolution out[l] = ifft(fft(in[l], n) * m)[:out_len]
    of a[nlines][in_len] into out[nlines][out_len] (dfft_lines_plan_create_convolve_padded_1d), which also takes lines longer
    than one shared-memory line.  `real_padded=(in_len, out_len)` with one_d instead: the same for real lines,
    out[l] = irfft(rfft(in[l], n) * m, n)[:out_len] (m: [n//2+1] per line; dfft_lines_plan_create_convolve_padded_r2c_1d)."""

    def __init__(self, three_d=None, precision=DOUBLE, real=False, flags=0, two_d=None, one_d=None, padded=None, real_padded=None):
        shapes = {"3d": three_d, "2d": two_d, "1d": one_d}
        given = [d for d, s in shapes.items() if s is not None]
        if len(given) != 1:
            raise ValueError("give exactly one of one_d, two_d and three_d")
        dims = given[0]
        if real_padded is not None:
            if dims != "1d" or real or padded is not None:
                raise ValueError("real_padded=(in_len, out_len) is a one_d plan, given without real=True and padded")
            n, nlines = one_d
            self._create("dfft_lines_plan_create_convolve_padded_r2c_1d", n, real_padded[0], real_padded[1], nlines, precision, flags)
            return
        if padded is not None:
            if dims != "1d" or real:
                raise ValueError("padded=(in_len, out_len) is a complex one_d plan")
            n, nlines = one_d
            self._create("dfft_lines_plan_create_convolve_padded_1d", n, padded[0], padded[1], nlines, precision, flags)
            return
        name = ("dfft_lines_plan_create_convolve_r2c_" if real else "dfft_lines_plan_create_convolve_") + dims
        self._create(name, *shapes[dims], precision, flags)

    def execute(self, in_ptr, out_ptr, mult_ptr, mult_count=1):
        _check(lib().dfft_lines_execute_convolve(self.handle, in_ptr, out_ptr, mult_ptr, mult_count), "dfft_lines_execute_convolve")


def _json_hook(fn, *args):
    """the JSON records of a host-only test hook that returns the bytes it needs for (buf, cap) = (None, 0), < 0 on error"""
    import json
    need = fn(*args, None, 0)
    if need < 0:
        raise DfftError(f"{fn.__name__} failed ({need}): " + lib().dfft_last_error().decode())
    buf = ctypes.create_string_buffer(int(need))
    fn(*args, buf, need)
    return json.loads(buf.value.decode())


def lines_conv_3d_ops(nx, ny, nz, batch, precision=DOUBLE, real=False, flags=0, mult_count=1):
    """passes LinesConvolvePlan(three_d=(nx, ny, nz, batch), ...) would launch per execute (host-only test hook, see
    dfft_debug_lines_conv_3d_ops; in = buffer 5, out = 2, temporary = 4, multiplier = 8); read DFFT_NO_PLANE /
    DFFT_FORCE_PLANE / DFFT_GENERIC at the call, as plan creation does"""
    return _json_hook(lib().dfft_debug_lines_conv_3d_ops, nx, ny, nz, batch, precision, int(bool(real)), flags, mult_count)


def lines_conv_2d_ops(nx, ny, batch, precision=DOUBLE, real=False, flags=0, mult_count=1):
    """passes LinesConvolvePlan(two_d=(nx, ny, batch), ...) would launch per execute (host-only test hook, see
    dfft_debug_lines_conv_2d_ops; buffers as lines_conv_3d_ops); read DFFT_NO_PLANE / DFFT_FORCE_PLANE / DFFT_GENERIC at the
    call, as plan creation does"""
    return _json_hook(lib().dfft_debug_lines_conv_2d_ops, nx, ny, batch, precision, int(bool(real)), flags, mult_count)


def lines_conv_1d_ops(n, nlines, precision=DOUBLE, real=False, flags=0, mult_count=1):
    """passes LinesConvolvePlan(one_d=(n, nlines), ...) would launch per execute (host-only test hook, see
    dfft_debug_lines_conv_1d_ops; buffers as lines_conv_3d_ops); read DFFT_GENERIC / DFFT_VARIANT at the call, as plan creation
    does"""
    return _json_hook(lib().dfft_debug_lines_conv_1d_ops, n, nlines, precision, int(bool(real)), flags, mult_count)


def lines_conv_padded_1d_ops(n, in_len, out_len, nlines, precision=DOUBLE, flags=0, mult_count=1, real=False):
    """passes LinesConvolvePlan(one_d=(n, nlines), padded=(in_len, out_len), ...) would launch per execute (host-only test hook,
    see dfft_debug_lines_conv_padded_1d_ops; buffers as lines_conv_3d_ops, temporary = 4); read DFFT_GENERIC / DFFT_VARIANT at
    the call, as plan creation does.  real=True: those of real_padded=(in_len, out_len) (dfft_debug_lines_conv_padded_r2c_1d_ops)"""
    fn = lib().dfft_debug_lines_conv_padded_r2c_1d_ops if real else lib().dfft_debug_lines_conv_padded_1d_ops
    return _json_hook(fn, n, in_len, out_len, nlines, precision, flags, mult_count)


def real_lines_ops(n, nlines, direction, precision=DOUBLE, two_d=None):
    """passes a RealLinesPlan(n, nlines, precision, two_d) would launch for `direction` (host-only test hook, see
    dfft_debug_real_lines_ops)"""
    args = (two_d[0], two_d[1], two_d[2], precision, direction, 1) if two_d is not None else (n, 1, nlines, precision, direction, 0)
    return _json_hook(lib().dfft_debug_real_lines_ops, *args)


def lines_3d_ops(nx, ny, nz, batch, direction, precision=DOUBLE, real=False):
    """passes LinesPlan(three_d=...) / RealLinesPlan(three_d=...) would launch for `direction` (host-only test hook, see
    dfft_debug_lines_3d_ops); read DFFT_NO_PLANE / DFFT_FORCE_PLANE / DFFT_GENERIC at the call, as plan creation does"""
    return _json_hook(lib().dfft_debug_lines_3d_ops, nx, ny, nz, batch, precision, direction, int(bool(real)))


def lines_ops(n, stride, nlines, inner, inner_dist, outer_dist, direction, precision=DOUBLE, two_d=False):
    """passes a lines plan would launch (host-only test hook, see dfft_debug_lines_ops)"""
    return _json_hook(lib().dfft_debug_lines_ops, n, stride, nlines, inner, inner_dist, outer_dist, precision, direction, int(two_d))


def _debug_op(rec):
    d = _DebugOp()
    for k in ("N", "C", "G", "W", "ntiles", "inv", "do_scale", "scale", "tw_n"):
        setattr(d, k, rec[k])
    d.in_, d.out, d.mult = rec.get("in") or None, rec.get("out") or None, rec.get("mult") or None
    d.ia[:], d.oa[:] = rec["ia"], rec["oa"]
    for side in ("ci", "co"):
        if side in rec:
            ch, dst = rec[side], getattr(d, side)
            dst.ediv, dst.nchunks = ch["ediv"], ch["nchunks"]
            for q in range(min(ch["nchunks"], 32)):
                dst.cptr[q], dst.SAq[q] = ch["cptr"][q] or None, ch["SAq"][q]
    return d


def debug_launch_op(rec, precision, second=None):
    """launch the kernel of one recorded pass (a dict of Plan.recorded_ops() with device pointers in place of its symbolic
    addresses) once on the current device and wait for it; a fused pair passes its second record as `second` (test hook
    dfft_debug_launch_op).  Returns the library's code: 0, or DFFT_EINVAL (-1) / DFFT_EUNSUPPORTED (-3) for a record it refuses."""
    a = _debug_op(rec)
    b = _debug_op(second) if second is not None else None
    return lib().dfft_debug_launch_op(rec["op"].encode(), ctypes.byref(a), second["op"].encode() if b is not None else None,
                                      ctypes.byref(b) if b is not None else None, precision)


def fft_lines(ptr, n, stride, nlines, inner, inner_dist, outer_dist, direction, precision=DOUBLE):
    _check(lib().dfft_fft_lines(ptr, n, stride, nlines, inner, inner_dist, outer_dist, direction, precision), "dfft_fft_lines")
