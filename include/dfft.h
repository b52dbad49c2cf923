/*
 * dfft.h -- C ABI of the H100-native slab-decomposed 3-D complex-to-complex FFT (libdfft.so), with real-to-complex /
 * complex-to-real plans over the same slabs (dfft_plan_r2c_3d).
 *
 * This is the drop-in boundary for the hot path of lueelu/DistributedFFT's `3dmpifft_opt`:
 * every entry point below names the reference interface it replaces (paths relative to the
 * reference tree).  Plain pointers and sizes only; all functions return 0 on success and a
 * negative DFFT_E* code on failure (dfft_last_error() gives the message).  The reference aborts
 * with exit(EXIT_FAILURE) on every error (3dmpifft_opt/include/fft_mpi_common.h:31-102); the C++
 * shim include/fft_mpi_3d_api.h keeps that behaviour on top of this ABI.
 *
 * Data model (identical to the reference, SURVEY.md Appendix A):
 *   global array A[x][y][z], z fastest, N0 = X slowest; P devices; device p owns the x-slab
 *   [p*xd, p*xd + n0_l), xd = ceil(N0/P), the last device the remainder.
 *   forward : in = natural x-slab [x_l][y][z]  ->  out = y-slab, TRANSPOSED [y_l][z][x] (x fastest)
 *   backward: in = [y_l][z][x]                 ->  out = natural [x_l][y][z], unnormalised.
 *   complex = interleaved (re, im) doubles (precision 0) or floats (precision 1).
 *
 * Threading: a plan belongs to one device; one host thread per device may create/execute plans
 * concurrently (the reference's `#pragma omp parallel for num_threads(devices)` loop,
 * 3dmpifft_opt/fftSpeed3d_c2c.cpp:49), or one process per device (torchrun) with a bootstrap
 * callback.  Collective calls (plan creation with P > 1, execute with P > 1, destroy) must be made
 * by all P participants.
 */
#ifndef DFFT_H
#define DFFT_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DFFT_FORWARD 1      /* fft_mpi_common.h:18 FORWARD  */
#define DFFT_BACKWARD (-1)  /* fft_mpi_common.h:19 BACKWARD */
#define DFFT_ALLOC_CPU 1    /* fft_mpi_common.h:15 ALLOC_CPU (pinned host memory here) */
#define DFFT_ALLOC_DEV (-1) /* fft_mpi_common.h:16 ALLOC_DEV */

#define DFFT_DOUBLE 0
#define DFFT_FLOAT 1

/* plan flags */
#define DFFT_EXCHANGE_AUTO 0u    /* P2P when every peer is reachable, else NCCL */
#define DFFT_EXCHANGE_P2P 1u     /* t1+t2 fused: the Y pass stores straight into the peers' receive buffers over NVLink */
#define DFFT_EXCHANGE_NCCL 2u    /* Y pass packs locally, grouped ncclSend/ncclRecv (ncclAlltoAll when the library has it) */
#define DFFT_EXCHANGE_STAGED 3u  /* reference-like: separate pack kernel + peer copies, device sync after every stage */
#define DFFT_EXCHANGE_MASK 3u
#define DFFT_SCALE_BACKWARD 4u   /* divide by N0*N1*N2 in the last backward pass (the `roc` variant's scale_element,
                                    3dmpifft_roc/include/fft_mpi_3d_api.cpp:208-210); default off like 3dmpifft_opt */

#define DFFT_NO_FUSE 8u          /* t0 as two HBM sweeps (Z pass, Y pass) */
#define DFFT_FORCE_FUSE 16u      /* t0 as ONE persistent kernel whose Z->Y intermediate stays in L2 (square planes only).
                                    Default: fused when the exchange is P2P (the Y stores are NVLink-bound and hide the
                                    Z role), and for one-device forward plans whose axis length has the TMA-pipelined fused
                                    kernel (512-point fp64); two sweeps otherwise.  Forced fusion of a one-device forward
                                    plan uses the TMA-pipelined kernel where it exists */

#define DFFT_NATURAL_SPECTRUM 64u /* single device: the spectrum (forward output / backward input) is kept in natural
                                    [x][y][z] order instead of the reference's transposed [y][z][x] (SURVEY 8f rank 1) */
#define DFFT_DRY_RUN 128u         /* describe-only plan (tests): no CUDA call, `in`/`out` are symbolic addresses, dfft_execute records
                                    the passes it would launch; read them with dfft_debug_plan_ops.  `comm` may be NULL */
#define DFFT_OVERLAP_X 32u       /* EXPERIMENTAL (forward, P2P, square planes): the whole transform of a device as one kernel;
                                    the z axis is sent in parts and the X lines of a part start as soon as it has arrived
                                    from every sender, overlapping t3 with the NVLink-bound sends (env DFFT_OVERLAP=1) */

#define DFFT_NO_PIPELINE 256u     /* P > 1: do NOT cut the z axis into parts.  Pipelined plans overlap t2 / t3 with t0 -- the reference has no
                                    overlap at all (fft_mpi_3d_api.cpp:610-672).  Two schedules exist: a CHAIN of two-role kernels on
                                    the plan stream, [Z + Y part 0] [Y part 1 + X part 0] ... [X last part] (forward, cubes, P2P
                                    exchange), and a TWO-STREAM schedule (send side / receive side, any direction, P2P or NCCL).
                                    Default (measured, DESIGN.md 5.1): the chain, from 4 devices on, for axes >= 1024 points.
                                    env DFFT_PIPELINE=0 / 1 overrides, DFFT_PARTS=k picks the number of parts,
                                    DFFT_PIPE_MODE=streams prefers the two-stream schedule */
#define DFFT_FORCE_PIPELINE 1024u /* pipelined plan wherever one is possible (also 2 devices, short axes, backward, NCCL with equal chunks) */

#define DFFT_NO_TMA 512u          /* use the register-staged pass kernels everywhere.  Default: passes whose load and store are both
                                    local and un-chunked (Z, natural Y, X) run on the TMA-pipelined kernels (fft_tma.cuh: 3-slot
                                    shared-memory ring fed and drained by cp.async.bulk / cp.async.bulk.tensor) for the lengths
                                    that have an instantiation; env DFFT_TMA=0 has the same effect.  TMA needs 16-byte-aligned
                                    addresses: a float plan whose bufferDev2 (`out`, or `in` in place) is only 8-byte aligned
                                    gets no TMA kernel either (a double plan with such a buffer is rejected, DFFT_EINVAL) */

#define DFFT_EINVAL (-1)
#define DFFT_ECUDA (-2)
#define DFFT_EUNSUPPORTED (-3)
#define DFFT_ECOMM (-4)
#define DFFT_ENOMEM (-5)

typedef struct dfft_plan_s* dfft_plan;
typedef struct dfft_comm_s* dfft_comm;

/* Bootstrap all-gather supplied by the host program in process-per-GPU mode: every rank
 * contributes `bytes` bytes from `send`; on return `recv` holds nranks*bytes in rank order.
 * Plays the role MPI_Comm plays in the reference (fft_mpi_3d_api.h:68,70). */
typedef int (*dfft_allgather_fn)(void* ctx, const void* send, void* recv, size_t bytes);

/* -- library ------------------------------------------------------------------------------- */
const char* dfft_last_error(void);
int dfft_version(void);
/* 2: `n` has a tuned kernel; 1: handled by the run-time-scheduled kernel (any length whose prime factors are
 * in {2,3,5,7,11,13} -- the set templateFFT accepts, templateFFT.cpp:3956-3964 -- up to 6400 points in double and
 * 12800 in float, i.e. while two copies of a line fit in shared memory); 0: unsupported (other primes, or longer:
 * the reference switches to multi-upload passes there, templateFFT.cpp:4007-4106, which this library does not have) */
int dfft_length_kind(int n, int precision);
/* radix schedule used for length n (stage order as executed); returns the number of stages, 0 if unsupported */
int dfft_length_schedule(int n, int precision, int* radices, int max_radices);
/* test hook (host only): ticket order of the single-kernel forward path (fft_fused3_kernel); out = role (0 Z, 1 Y, 2 X),
 * part, plane, tile; returns the number of tickets (ticket < 0: only that) */
long long dfft_debug_fused3_order(long long planes, long long rows, int GA, int GBk, int GXk, int K, int lag, long long ticket,
                                  long long out[4]);
/* test hook (host only): ticket order of the two-role t0 kernels (fft_fused2_kernel, fft_tma_fused_zy_kernel); out = role
 * (0 first role, 1 second role), plane, tile; returns the number of tickets (ticket < 0: only that) */
long long dfft_debug_fused2_order(long long planes, int GA, int GB, int lag, long long ticket, long long out[3]);
/* test hook: JSON description of the passes recorded by the last dfft_execute of a DFFT_DRY_RUN plan (affine maps, chunk
 * tables, symbolic buffer addresses: device d, buffer b at ((d+1) << 44) | (b << 40), b = 1 bufferDev1, 2 out, 3 receive/work,
 * 4 intermediate, 5 in).  Returns the number of bytes needed (including the terminator). */
long long dfft_debug_plan_ops(dfft_plan plan, char* buf, long long cap);
/* test hook: one record of dfft_debug_plan_ops with its symbolic addresses replaced by device pointers.  A side without a chunk
 * table has nchunks = 0; `mult` is the multiplier of an "XCONV" / "XCONV_CO" record, NULL otherwise. */
typedef struct dfft_debug_chunks {
    int ediv, nchunks;
    void* cptr[32];       /* at most 32 chunks, one per device */
    long long SAq[32];
} dfft_debug_chunks;
typedef struct dfft_debug_op {
    int N, C, G, W;
    long long ntiles;
    int inv, do_scale;
    double scale;
    long long tw_n;
    void *in, *out, *mult;
    long long ia[4], oa[4];
    dfft_debug_chunks ci, co;
} dfft_debug_op;
/* test hook: launch the kernel of one record once on the current device's legacy default stream and wait for it, with the
 * twiddle table its entry and kind use in a plan and no arrival flags (nothing waits, nothing is signalled).  `op` is the
 * record's name: "Z", "Y", "Y_CO", "Y_CI", "XF", "XB", "XB_CO", "XF_TW", "XCONV", "XCONV_CO", or the first record of a fused
 * pair ("fusedZ" forward, "fusedY" backward) with the other record and its name in `second` / `second_op` (NULL otherwise); a
 * pair runs as one two-role kernel on its own zeroed plane counters.  Plans never call it.  DFFT_EINVAL: an unknown name, a single-kernel forward
 * record ("ovlZ" / "ovlY" / "ovlX"), a C other than the entry's for that kind, inconsistent tiling, a missing or superfluous
 * chunk table, a null pointer, a bad precision; DFFT_EUNSUPPORTED: the entry has no such kernel. */
int dfft_debug_launch_op(const char* op, const dfft_debug_op* rec, const char* second_op, const dfft_debug_op* second, int precision);
/* test hook (host only): the passes a lines plan (1-D, 2-D when two_d != 0: n = nx, stride = ny, nlines = batch, or the
 * four-step plan of a long line) would launch, same JSON as dfft_debug_plan_ops: data = buffer 1, temporary = buffer 4 */
long long dfft_debug_lines_ops(int n, long long stride, long long nlines, long long inner, long long inner_dist, long long outer_dist,
                               int precision, int direction, int two_d, char* buf, long long cap);
/* number of TUNED transform lengths for a precision; fills `lengths` (may be NULL) */
int dfft_supported_lengths(int precision, int* lengths, int max_lengths);

/* -- slab bookkeeping ---------------------------------------------------------------------- */
/* fft_mpi_init, fft_mpi_3d_api.cpp:3-39 (+ getProperDeviceNum :232-272, getDataCountForNode :274-287):
 * shrink `wanted_devices` (clamped to the visible device count unless that is 0) so that ceil-blocks
 * of N[0] leave no device empty, return per-device input element counts, enable peer access
 * between the devices used.  `counts` must have room for `wanted_devices` entries. */
int dfft_init(const long long N[3], int wanted_devices, int* total_devices, int* local_devices, long long* counts);
/* getMaxDataCount, fft_mpi_3d_api.cpp:289-316: elements each of in/out must hold on a device */
long long dfft_max_data_count(long long n0, long long n1, long long n2, int total_devices, int is_last_device);
/* fft_mpi_local_size_3d (declared fft_mpi_3d_api.h:73, never defined in the reference): returns the
 * allocation count and the slab owned by `dev_idx` before (x) and after (y) the exchange */
long long dfft_local_size_3d(long long n0, long long n1, long long n2, int total_devices, int dev_idx,
                             long long* local_n0, long long* local_0_start, long long* local_n1,
                             long long* local_1_start);
/* fft_mpi_alloc_local_memory, fft_mpi_3d_api.cpp:216-230 (64-bit count; ALLOC_CPU is pinned) */
void* dfft_alloc_local(long long count, int flag, int precision);
int dfft_free_local(void* ptr, int flag);

/* -- communicator -------------------------------------------------------------------------- */
/* P device-threads inside one process (the reference's multi-GPU-per-rank mode). Returns one shared
 * handle; every participating thread passes it to dfft_plan_c2c_3d with its own dev_idx. */
int dfft_comm_create_local(int nranks, dfft_comm* comm);
/* One process per GPU; `allgather` is used during plan creation / teardown only. */
int dfft_comm_create_bootstrap(int rank, int nranks, dfft_allgather_fn allgather, void* ctx, dfft_comm* comm);
int dfft_comm_destroy(dfft_comm comm);
/* host-side all-gather through a communicator (what plan creation uses to swap IPC handles / the NCCL id) */
int dfft_comm_allgather(dfft_comm comm, int rank, const void* send, void* recv, size_t bytes);
/* the reference's TransInfo exchange table of one device (fft_mpi_common.h:24-29, fft_mpi_3d_api.cpp:84-133):
 * element counts and offsets of the chunk sent to / received from every device i */
int dfft_exchange_table(long long n0, long long n1, long long n2, int total_devices, int dev_idx, int direction,
                        long long* scount, long long* soffset, long long* rcount, long long* roffset);

/* -- plan / execute ------------------------------------------------------------------------ */
/* fft_mpi_plan_dft_c2c_3d, fft_mpi_3d_api.cpp:41-141.  Same ownership rules: `in`/`out` are the
 * caller's device buffers of dfft_max_data_count() elements; out == NULL or out == in means in
 * place; the plan owns bufferDev1 and copies `in` into it at creation (api.cpp:76-77); bufferDev2
 * aliases `out`.  Execute never re-reads `in`: refill bufferDev1 (dfft_plan_buffers) to transform new
 * data, exactly like the reference driver does (fftSpeed3d_c2c.cpp:78).
 * `comm` may be NULL when total_devices == 1.  `dev_idx` is this device's global index (= rank).
 * The CUDA device current at the call is the plan's device. */
int dfft_plan_c2c_3d(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                     int total_devices, int direction, int precision, unsigned flags, dfft_plan* plan);
/* Real-to-complex (direction DFFT_FORWARD) and complex-to-real (DFFT_BACKWARD) transforms over the same slabs.
 * R2C: in = real x-slab [x_l][y][z] (n0_l*n1*n2 reals) -> out = half spectrum, the C2C forward layout with z cut to
 *      nzh = n2/2 + 1: [y_l][nzh][x] (x fastest), or [x][y][nzh] with DFFT_NATURAL_SPECTRUM (one device).
 * C2R: the exact inverse layout, unnormalised (DFFT_SCALE_BACKWARD: 1/(n0*n1*n2)).  Any complex input is accepted and the
 *      result is numpy.fft.irfftn(., s=(n0,n1,n2)) * n0*n1*n2: the imaginary parts at z = 0 and z = n2/2 (even n2) of every
 *      z-line are ignored, as FFTW and numpy do.
 * The buffers hold exactly dfft_local_size_r2c_3d()'s counts (reals on the real side, complex elements on the other); the
 * plan never touches anything past them and copies `in` into its bufferDev1 at creation like the C2C plan.  `out` must be a
 * separate buffer (NULL or out == in: DFFT_EINVAL).  The z length needs a tuned kernel (dfft_length_kind(n2, precision) == 2);
 * y and x may be any length the C2C plan accepts.  Every device count and the P2P / NCCL exchanges work; DFFT_EXCHANGE_STAGED
 * (and dfft_execute_stage) is DFFT_EUNSUPPORTED.  The fusion / overlap / pipeline flags are accepted and have no effect.
 * dfft_plan_counts gives in_count / out_count in elements of their own type. */
int dfft_plan_r2c_3d(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                     int total_devices, int direction, int precision, unsigned flags, dfft_plan* plan);
/* element counts of one device: reals of its x-slab, complex elements of its half-spectrum slab */
int dfft_local_size_r2c_3d(long long n0, long long n1, long long n2, int total_devices, int dev_idx,
                           long long* real_count, long long* complex_count);
/* Spectral convolution plans: forward transform, pointwise multiply, inverse transform in one plan, with the multiply folded into
 * one x-column pass (forward FFT along x, multiply, inverse FFT along x) so the spectrum never reaches memory in transposed order.
 *   C2C: out = IFFT3( m .* FFT3(in) ), unnormalised (x n0*n1*n2) unless DFFT_SCALE_BACKWARD.
 *   R2C: out = irfftn( m .* rfftn(in), s=(n0,n1,n2) ) * n0*n1*n2 (numpy's C2R convention), real in / real out.
 * `in` and `out` are this device's x-slab [x_l][y][z], exactly local_n0*n1*n2 elements (complex for C2C, reals for R2C); the plan
 * never touches anything past them.  Ownership as for the other plans: `in` is snapshotted into bufferDev1 at creation and every
 * execute transforms that snapshot (refill it through dfft_plan_buffers for new data; it is never written); out == NULL or
 * out == in means in place; creation, execute and destroy are collective when P > 1.
 * The multiplier is given at each execute (one plan serves many multipliers): read-only, complex in the plan's precision, aligned to
 * its element size, in NATURAL order over this device's y-slab: m[x][y_l][z'], x < n0, y_l < local_n1 starting at local_1_start
 * (dfft_local_size_3d), z' < n2 (C2C) or n2/2+1 (R2C).  With one device that is the natural [x][y][z] array.
 * Flags: DFFT_SCALE_BACKWARD, DFFT_EXCHANGE_AUTO / P2P / NCCL and DFFT_DRY_RUN (the multiplier is then a symbolic address too)
 * are honoured; DFFT_NO_TMA, DFFT_NO_FUSE and DFFT_FORCE_FUSE select the forward and the backward t0 exactly as for C2C plans of
 * the same shape; the pipeline and overlap flags are accepted and have no effect.
 * DFFT_EUNSUPPORTED: DFFT_EXCHANGE_STAGED; an x length without a tuned kernel (dfft_length_kind(n0, precision) != 2) or a
 * DFFT_VARIANT entry without the convolution kernels; y / z lengths the C2C (R2C) plan rejects.
 * DFFT_EINVAL: DFFT_NATURAL_SPECTRUM (no spectrum is exposed); dfft_execute, dfft_execute_stage and dfft_execute_host* on a
 * convolve plan; dfft_execute_convolve on any other plan; a null or misaligned multiplier.
 * dfft_get_timings after dfft_execute_convolve: t[0] = forward half (its t0 and, P > 1, its exchange), t[1] = 0, t[2] = backward
 * half (its exchange and t0), t[3] = the fused X pass, t[4] = total. */
int dfft_plan_convolve_c2c_3d(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                              int total_devices, int precision, unsigned flags, dfft_plan* plan);
int dfft_plan_convolve_r2c_3d(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                              int total_devices, int precision, unsigned flags, dfft_plan* plan);
/* Asynchronous on the plan's stream, like dfft_execute; result in bufferDev2 (= out) */
int dfft_execute_convolve(dfft_plan plan, const void* multiplier);
/* fft_mpi_execute_dft_3d_c2c, fft_mpi_3d_api.cpp:181-214.  Asynchronous on the plan's stream;
 * dfft_synchronize() or dfft_get_timings() waits.  Result in bufferDev2 (= out). */
int dfft_execute(dfft_plan plan);
int dfft_synchronize(dfft_plan plan);
/* One reference stage at a time (0: t0 fftZY, 1: t1 pack, 2: t2 all-to-all, 3: t3 fftX, in the
 * order the plan's direction executes them), leaving bufferDev1/bufferDev2 exactly as the reference
 * leaves them after that stage.  Requires a plan created with DFFT_EXCHANGE_STAGED.  Synchronous. */
int dfft_execute_stage(dfft_plan plan, int stage);
/* Host-buffer entry: copies `host_in` (input-slab elements) to bufferDev1, executes, copies the
 * result slab to `host_out`; copies are on the plan's stream (pinned buffers overlap). Synchronous. */
int dfft_execute_host(dfft_plan plan, const void* host_in, void* host_out);
/* Same, but returns once the three operations are enqueued on the plan's stream (dfft_synchronize waits).
 * Two plans driven alternately keep PCIe busy in both directions: plan A's D2H overlaps plan B's H2D. */
int dfft_execute_host_async(dfft_plan plan, const void* host_in, void* host_out);
/* milliseconds of the last execute: t[0..3] = t0,t1,t2,t3 as the reference prints them
 * (api.cpp:201; fused stages report 0 for t1 and the *exposed* wait for t2), t[4] = total. */
int dfft_get_timings(dfft_plan plan, double t_ms[5]);
/* milliseconds of the Z, Y and X pass kernels of the last execute (CUDA events around each launch) */
int dfft_get_pass_timings(dfft_plan plan, double t_ms[3]);
/* bufferDev1 / bufferDev2 of the plan (fft_mpi_3d_api.h:24; the driver writes into bufferDev1) */
int dfft_plan_buffers(dfft_plan plan, void** buffer1, void** buffer2);
/* element counts of this device's input slab and output slab */
int dfft_plan_counts(dfft_plan plan, long long* in_count, long long* out_count, long long* max_count);
/* kernels launched by the last execute (for bench.py's gpu_launches) */
int dfft_plan_launches(dfft_plan plan);
/* 2: forward transform runs as the single overlapped kernel (DFFT_OVERLAP_X); 1: t0 runs as the fused two-pass
 * kernel (square planes, N1 == N2); 0: separate passes */
int dfft_plan_fused(dfft_plan plan);
/* bit 0 / 1 / 2 set: the plan's un-chunked Z / Y / X pass runs on the TMA-pipelined kernel (fft_tma.cuh) */
int dfft_plan_tma_mask(dfft_plan plan);
/* developer hook: device-side timeline of the last execute of a DFFT_OVERLAP_X plan created under DFFT_DEBUG_TIMELINE=1 (microseconds
 * from kernel start: end of phase 0, first X tile, kernel end; mean us per Z / Y / X tile; tile counts; mean / max arrival wait) */
int dfft_debug_timeline(dfft_plan plan, double out[11]);
/* number of z-parts of the stream-pipelined forward / backward path, 0 when the plan does not use it */
int dfft_plan_pipeline_parts(dfft_plan plan);
/* 1: the z-parts of a pipelined forward plan run as a chain of two-role kernels on one stream (Y pass of part k + X pass of
 * part k-1 in one kernel: cubes with the P2P exchange), 0: as two streams, or not pipelined */
int dfft_plan_pipeline_chain(dfft_plan plan);
/* which exchange the plan resolved to (DFFT_EXCHANGE_*) */
int dfft_plan_exchange(dfft_plan plan);
/* the stream the plan launches on (a cudaStream_t), so callers can time with events on it */
void* dfft_plan_stream(dfft_plan plan);
/* fft_mpi_destroy_plan, fft_mpi_3d_api.cpp:143-179 (collective when P > 1) */
int dfft_destroy(dfft_plan plan);
/* fft_mpi_cleanup (declared fft_mpi_3d_api.h:69, never defined in the reference) */
int dfft_cleanup(void);

/* convenience for hosts without a CUDA runtime binding (tests): synchronous cudaMemcpy,
 * kind 1 = host->device, 2 = device->host, 0 = default (UVA) */
int dfft_memcpy(void* dst, const void* src, size_t bytes, int kind);

/* -- batched local transforms: the templateFFT engine surface (3dmpifft_opt/include/templateFFT.h:361-365) -----
 *    initializeFFT(app, config)   -> dfft_lines_plan_create / dfft_lines_plan_create_2d
 *    launchFFTKernel(app, inverse)-> dfft_lines_execute (asynchronous on the plan's stream, in place)
 *    deleteFFT(app)               -> dfft_lines_destroy
 *    Line l starts at data + (l / inner) * outer_dist + (l % inner) * inner_dist (in elements), points are
 *    `stride` elements apart.  Supported shapes: stride == 1 with densely packed lines (inner_dist == n), or
 *    stride > 1 with inner_dist == 1 (columns of row-major matrices: `inner` columns per matrix, matrices
 *    `outer_dist` apart; padded rows, gaps between matrices and interleaved matrices are fine).  Columns must not
 *    overlap: the (extent, stride) pairs (inner, 1), (n, stride) and (nlines / inner, outer_dist), sorted by stride,
 *    each need a stride at least the span of the ones before ((extent - 1) * stride summed, plus one); pairs of
 *    extent 1 are left out, so a single matrix (nlines == inner) ignores outer_dist.  An overlapping layout, or a
 *    negative outer_dist over two or more matrices, is DFFT_EINVAL.  The elements between columns and matrices are
 *    never read or written.  The 2-D plan transforms `batch` row-major ny x nx matrices (nx fastest), the
 *    reference's FFTdim = 2 application (templateFFT/batchTest/Test_2D.cpp). */
typedef struct dfft_lines_plan_s* dfft_lines_plan;
int dfft_lines_plan_create(int n, long long stride, long long nlines, long long inner, long long inner_dist,
                           long long outer_dist, int precision, dfft_lines_plan* plan);
int dfft_lines_plan_create_2d(int nx, int ny, long long batch, int precision, dfft_lines_plan* plan);
/* batch row-major nz x ny x nx complex arrays (nx fastest), in place through dfft_lines_execute:
 * numpy.fft.fftn(a, axes=(1, 2, 3)) on a[batch][nz][ny][nx]; backward unnormalised (ifftn * nx*ny*nz).
 * nx takes any length a contiguous lines pass takes, ny and nz any length a strided one takes.  Where nx == ny is 16, 32 or 64
 * the X and Y passes run as one kernel over whole planes held in shared memory (DFFT_NO_PLANE=1 at plan creation: separate
 * passes; the results are bitwise the same).  2^31 or more rows (ny*nz*batch) are DFFT_EUNSUPPORTED. */
int dfft_lines_plan_create_3d(int nx, int ny, int nz, long long batch, int precision, dfft_lines_plan* plan);
int dfft_lines_execute(dfft_lines_plan plan, void* data, int direction);
int dfft_lines_synchronize(dfft_lines_plan plan);
void* dfft_lines_stream(dfft_lines_plan plan);
int dfft_lines_destroy(dfft_lines_plan plan);
/* Real-data lines (R2C forward / C2R backward), out of place, on the same engine:
 *    1-D: nlines densely packed real lines of n points  <->  nlines densely packed half spectra of n/2+1 complex points.
 *    2-D: batch row-major ny x nx real matrices (nx fastest)  <->  batch ny x (nx/2+1) complex matrices (numpy.fft.rfft2 layout).
 * The real axis (n, nx) takes every length with dfft_length_kind(n, precision) >= 1: tuned lengths run on the real kernels of
 * the 3-D plan's Z pass, other 2..13-smooth lengths up to one shared-memory line on the run-time-scheduled real kernels.  Longer
 * lines, other prime factors, n < 2, a DFFT_VARIANT kernel entry without real kernels and 2^31 or more real lines are
 * DFFT_EUNSUPPORTED.  The 2-D plan's ny takes any length a strided C2C lines pass takes; its backward transform uses a
 * plan-owned temporary of batch*ny*(nx/2+1) complex elements. */
int dfft_lines_plan_create_r2c(int n, long long nlines, int precision, dfft_lines_plan* plan);
int dfft_lines_plan_create_r2c_2d(int nx, int ny, long long batch, int precision, dfft_lines_plan* plan);
/* batch real nz x ny x nx arrays <-> batch nz x ny x (nx/2+1) complex arrays (numpy.fft.rfftn layout), out of place through
 * dfft_lines_execute_real; C2R = irfftn(., s=(nz, ny, nx)) * nx*ny*nz, with the same ignored imaginary parts as the 2-D C2R.
 * nx as the 1-D real plan, ny and nz as a strided C2C lines pass; the backward transform uses a plan-owned temporary of
 * batch*nz*ny*(nx/2+1) complex elements and never writes `in`.  2^31 or more real rows are DFFT_EUNSUPPORTED. */
int dfft_lines_plan_create_r2c_3d(int nx, int ny, int nz, long long batch, int precision, dfft_lines_plan* plan);
/* FORWARD: in = reals -> out = half spectra.  BACKWARD: in = half spectra -> out = reals, unnormalised (numpy.fft.irfft / irfft2
 * times n / nx*ny; the imaginary parts at bin 0 and, for even n, bin n/2 are ignored, as in the 3-D C2R).  `in` is never
 * written.  Null or overlapping buffers, a buffer not aligned to its element size, and a complex plan are DFFT_EINVAL (and a
 * real plan passed to dfft_lines_execute).  Asynchronous on the plan's stream (dfft_lines_synchronize waits). */
int dfft_lines_execute_real(dfft_lines_plan plan, const void* in, void* out, int direction);
/* test hook (host only): the passes of a real lines plan (1-D: n, nlines = batch, ny unused; 2-D when two_d != 0), same JSON
 * as dfft_debug_lines_ops, with "nzh" and "pair" on the real passes; in = buffer 5, out = buffer 2, temporary = buffer 4 */
long long dfft_debug_real_lines_ops(int n, int ny, long long batch, int precision, int direction, int two_d, char* buf, long long cap);
/* test hook (host only): the passes of either 3-D lines plan for `direction`, JSON like dfft_debug_lines_ops (complex, data =
 * buffer 1) / dfft_debug_real_lines_ops (real != 0); the plane kernel is one "XY_PLANE" record over ntiles planes */
long long dfft_debug_lines_3d_ops(int nx, int ny, int nz, long long batch, int precision, int direction, int real,
                                  char* buf, long long cap);
/* Batched 3-D spectral convolution on the lines engine: batch row-major nz x ny x nx volumes (nx fastest),
 *   C2C: out = ifftn(fftn(in) * m) over axes (1, 2, 3), unnormalised (x nx*ny*nz) unless DFFT_SCALE_BACKWARD;
 *   R2C: out = irfftn(rfftn(in) * m, s=(nz, ny, nx)) * nx*ny*nz, real in / real out (numpy's C2R convention, as
 *        dfft_plan_convolve_r2c_3d: the imaginary parts the C2R ignores are ignored here too).
 * m is complex in the plan's precision, natural order: [z][y][x] (C2C) or [z][y][nx/2+1] (R2C) per volume.  One execute runs
 * the forward passes of the 3-D lines plan with the Z pass replaced by one column pass that transforms along z, multiplies and
 * transforms back (the slab convolve plan's fused X pass), then the passes before it inverted: 3 launches where nx == ny has the
 * plane kernel of dfft_lines_plan_create_3d (read at creation, DFFT_NO_PLANE / DFFT_FORCE_PLANE as there), 5 otherwise.  The
 * R2C plan owns a temporary of batch*nz*ny*(nx/2+1) complex elements.
 * Lengths: nz needs a tuned kernel of the default table (dfft_length_kind(nz, precision) == 2; DFFT_GENERIC and DFFT_VARIANT
 * entries are DFFT_EUNSUPPORTED).  C2C: nx and ny as dfft_lines_plan_create_3d; R2C: nx as dfft_lines_plan_create_r2c_3d, ny as
 * a strided C2C lines pass.  2^31 or more rows are DFFT_EUNSUPPORTED, as in the 3-D lines plans.
 * Flags: DFFT_SCALE_BACKWARD folds 1/(nx*ny*nz) into the multiply; any other bit is DFFT_EINVAL. */
int dfft_lines_plan_create_convolve_3d(int nx, int ny, int nz, long long batch, int precision, unsigned flags, dfft_lines_plan* plan);
int dfft_lines_plan_create_convolve_r2c_3d(int nx, int ny, int nz, long long batch, int precision, unsigned flags, dfft_lines_plan* plan);
/* Batched 2-D spectral convolution on the lines engine: batch row-major ny x nx images (nx fastest),
 *   C2C: out = ifft2(fft2(in) * m), unnormalised (x nx*ny) unless DFFT_SCALE_BACKWARD;
 *   R2C: out = irfft2(rfft2(in) * m, s=(ny, nx)) * nx*ny, real in / real out (the imaginary parts the C2R ignores are ignored
 *        here too, as in the 3-D R2C convolve plan).
 * m is complex in the plan's precision, natural order: [y][x] (C2C) or [y][nx/2+1] (R2C) per image.  C2C with nx == ny of 16,
 * 32 or 64 runs the whole convolution in one kernel (X, Y, multiply, inverse Y, inverse X on images held in shared memory: 2
 * sweeps over the batch + the multiplier) where that kernel is the default for the shape (read at creation; DFFT_NO_PLANE=1
 * never uses it, DFFT_FORCE_PLANE=1 wherever it is instantiated).  Otherwise 3 launches: X, one column pass that transforms
 * along y, multiplies and transforms back, inverse X (R2C: the real row pass, the column pass over the nx/2+1 columns, the
 * inverse real row pass).  The R2C plan owns a temporary of batch*ny*(nx/2+1) complex elements.
 * Lengths: ny needs a tuned kernel of the default table (dfft_length_kind(ny, precision) == 2; DFFT_GENERIC and DFFT_VARIANT
 * entries are DFFT_EUNSUPPORTED).  nx: C2C as dfft_lines_plan_create_2d, R2C as dfft_lines_plan_create_r2c_2d.  2^31 or more
 * rows (ny*batch) are DFFT_EUNSUPPORTED.
 * Flags: DFFT_SCALE_BACKWARD folds 1/(nx*ny) into the multiply; any other bit is DFFT_EINVAL.  Executed with
 * dfft_lines_execute_convolve, under the same rules as the 3-D plans. */
int dfft_lines_plan_create_convolve_2d(int nx, int ny, long long batch, int precision, unsigned flags, dfft_lines_plan* plan);
int dfft_lines_plan_create_convolve_r2c_2d(int nx, int ny, long long batch, int precision, unsigned flags, dfft_lines_plan* plan);
/* Batched 1-D spectral convolution on the lines engine: nlines densely packed lines of n points,
 *   C2C: out = ifft(fft(in) * m) per line, unnormalised (x n) unless DFFT_SCALE_BACKWARD;
 *   R2C: out = irfft(rfft(in) * m, n) * n, real in / real out (the imaginary parts of m[0] and, for even n, m[n/2] are ignored,
 *        numpy's C2R convention, as in the 2-D and 3-D R2C convolve plans).
 * m is complex in the plan's precision: [n] (C2C) or [n/2+1] (R2C) per line.  One execute is one launch that reads the batch
 * once, writes it once and reads the multiplier: forward transform, multiply and inverse transform of every line in registers
 * and shared memory (R2C: two real lines per complex transform).  No temporary.
 * Lengths: n needs a tuned kernel of the default table (dfft_length_kind(n, precision) == 2); generic lengths, DFFT_GENERIC and
 * DFFT_VARIANT entries and lines longer than one shared-memory line are DFFT_EUNSUPPORTED, as is R2C with n < 2.  2^31 or more
 * lines are DFFT_EUNSUPPORTED.  Flags: DFFT_SCALE_BACKWARD folds 1/n into the multiply; any other bit is DFFT_EINVAL.  Executed
 * with dfft_lines_execute_convolve (batch = nlines), under the same rules as the 2-D and 3-D plans.  Longer lines, and linear
 * (zero-padded) convolution, are dfft_lines_plan_create_convolve_padded_1d's. */
int dfft_lines_plan_create_convolve_1d(int n, long long nlines, int precision, unsigned flags, dfft_lines_plan* plan);
int dfft_lines_plan_create_convolve_r2c_1d(int n, long long nlines, int precision, unsigned flags, dfft_lines_plan* plan);
/* Batched zero-padded 1-D spectral convolution on the lines engine (C2C): `in` holds nlines densely packed lines of in_len points
 * (line l at l*in_len), `out` nlines lines of out_len points (line l at l*out_len), and per line
 *   out[l] = (ifft(fft(zero_pad(in[l], n)) * m_l))[0:out_len],
 * unnormalised (x n) unless DFFT_SCALE_BACKWARD.  With n >= in_len + K - 1 this is the linear convolution of a line with a filter of
 * K points whose n-point spectrum is m; in_len = out_len = n is the circular convolution of dfft_lines_plan_create_convolve_1d.
 * A shift of the output window is a phase ramp on m.  m is [n] complex in the plan's precision, natural order, per line or shared.
 * Two paths, chosen from n:
 *   n with a tuned kernel of the default table: one launch that reads in_len and writes out_len points per line; no temporary.
 *   n = n1 * n2 (n1 <= 2 sqrt(n)) of tuned lengths of the default table: three launches of the four-step transform (the padding
 *   folded into the first pass's loads and the last pass's stores, the multiply into the middle pass), with a temporary of
 *   nlines * n complex elements owned by the plan.  Lines of up to 4096 * 4096 = 2^24 points, and short untuned lengths that split so.
 * DFFT_EINVAL: in_len or out_len outside [1, n], n < 1, nlines < 0, a bad precision, any flag but DFFT_SCALE_BACKWARD, a null plan
 * pointer.  DFFT_EUNSUPPORTED: 2^31 or more lines, a length that takes neither path, DFFT_GENERIC and DFFT_VARIANT entries.
 * Executed with dfft_lines_execute_convolve (batch = nlines) under its rules; in == out is allowed only when in_len == out_len. */
int dfft_lines_plan_create_convolve_padded_1d(int n, long long in_len, long long out_len, long long nlines, int precision,
                                              unsigned flags, dfft_lines_plan* plan);
/* The same for real lines (R2C): `in` holds nlines densely packed real lines of in_len points, `out` nlines real lines of out_len
 * points, and per line
 *   out[l] = irfft(rfft(zero_pad(in[l], n)) * m_l, n)[0:out_len],
 * unnormalised (x n) unless DFFT_SCALE_BACKWARD.  m is [n/2 + 1] complex in the plan's precision, per line or shared; the
 * imaginary parts of m[0] and (even n) m[n/2] are ignored, as numpy's irfft ignores them.  Two real lines go through one complex
 * transform.  The same two paths and splits as the complex plan:
 *   n with a tuned kernel of the default table: one launch; no temporary.
 *   n = n1 * n2: three launches of the four-step transform over ceil(nlines / 2) complex lines, with a temporary of
 *   ceil(nlines / 2) * n complex elements owned by the plan; the middle pass finds each bin k and its mirror n - k in one tile.
 * DFFT_EINVAL as the complex plan.  DFFT_EUNSUPPORTED: n < 2, and as the complex plan.  Executed with dfft_lines_execute_convolve
 * (batch = nlines, real elements) under its rules; in == out is allowed only when in_len == out_len. */
int dfft_lines_plan_create_convolve_padded_r2c_1d(int n, long long in_len, long long out_len, long long nlines, int precision,
                                                  unsigned flags, dfft_lines_plan* plan);
/* mult_count = 1: one multiplier shared by every line / image / volume; = batch: one each, densely packed.  in == out (in place) or
 * disjoint buffers; `in` is never written when they are distinct, `mult` never.  DFFT_EINVAL: a null pointer, a buffer not
 * aligned to its element size (fp32 complex at an 8-byte offset is fine), a partial overlap of in and out (or in == out for a padded
 * plan whose in_len and out_len differ), a multiplier that
 * overlaps out, another mult_count, and a plan that is not a convolve lines plan (dfft_lines_execute / dfft_lines_execute_real
 * on a convolve plan are DFFT_EINVAL too).  Asynchronous on the plan's stream (dfft_lines_synchronize waits). */
int dfft_lines_execute_convolve(dfft_lines_plan plan, const void* in, void* out, const void* mult, long long mult_count);
/* test hook (host only): the passes of either convolve lines plan, JSON as dfft_debug_lines_3d_ops with in = buffer 5, out = 2,
 * temporary = 4, multiplier = 8; the column pass is "XCONV" with "mult" and "shared" (1 when mult_count == 1) */
long long dfft_debug_lines_conv_3d_ops(int nx, int ny, int nz, long long batch, int precision, int real, unsigned flags,
                                       long long mult_count, char* buf, long long cap);
/* the same for the 2-D convolve lines plans; the one-kernel convolution is one "XY_PLANE_CONV" record with ntiles = images,
 * ia = oa = [image, 0, row, point] strides, "mult" and "shared" */
long long dfft_debug_lines_conv_2d_ops(int nx, int ny, long long batch, int precision, int real, unsigned flags,
                                       long long mult_count, char* buf, long long cap);
/* the same for the 1-D convolve lines plans: one "LINE_CONV" record (real != 0: "LINE_CONV_R2C", which also carries "nzh" and
 * "pair" as the real lines records) with C lines (line pairs) per tile, ntiles = G tiles, W = nlines, "mult" and "shared" */
long long dfft_debug_lines_conv_1d_ops(int n, long long nlines, int precision, int real, unsigned flags, long long mult_count,
                                       char* buf, long long cap);
/* the same for the zero-padded 1-D convolve lines plans: one "LINE_CONV_PAD" record (short path) or "XF_TW_PAD", "XCONV" and
 * "XB_TW_PAD" (long path, temporary = buffer 4); the padded records carry "in_len" and "out_len" */
long long dfft_debug_lines_conv_padded_1d_ops(int n, long long in_len, long long out_len, long long nlines, int precision,
                                              unsigned flags, long long mult_count, char* buf, long long cap);
/* the same for the real zero-padded 1-D convolve lines plans: one "LINE_CONV_PAD_R2C" record (short path, C line pairs per tile)
 * or "XF_TW_PAD_R2C", "XCONV_R2C" and "XB_TW_PAD_C2R" (long path, temporary = buffer 4).  Every record carries "in_len", "out_len"
 * and "lines" (real lines); those that touch the real lines "pair" (the distance between a pair's two lines on the input / output
 * side, 0 on a complex side); LINE_CONV_PAD_R2C and XCONV_R2C "mult", "shared" and "nzh" (n/2 + 1) */
long long dfft_debug_lines_conv_padded_r2c_1d_ops(int n, long long in_len, long long out_len, long long nlines, int precision,
                                                  unsigned flags, long long mult_count, char* buf, long long cap);
/* one-shot convenience (plan + execute + synchronize + destroy), used by the per-axis parity tests */
int dfft_fft_lines(void* data, int n, long long stride, long long nlines, long long inner, long long inner_dist,
                   long long outer_dist, int direction, int precision);

#ifdef __cplusplus
}
#endif
#endif /* DFFT_H */
