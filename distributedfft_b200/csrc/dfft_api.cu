// dfft_api.cu -- C-ABI implementation: slab bookkeeping, communicator, plan, stage sequencing.
//
// Host-side counterpart of 3dmpifft_opt/include/fft_mpi_3d_api.cpp (plan :41-141, execute :181-214,
// stages :466-699) re-designed for the GPU: three batched pass launches per transform instead of two
// launches per plane, the pack folded into the Y-pass store, the all-to-all either fused into that
// store over NVLink peer mappings or handed to NCCL, CUDA events instead of host timers, explicit
// streams and no device-wide syncs on the production path.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cassert>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/dfft.h"
#include "dfft_kernels.cuh"
#include "fft_tma.cuh"

using namespace dfft;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static int fail(int code, const char* fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    if (getenv("DFFT_VERBOSE")) fprintf(stderr, "[dfft] error %d: %s\n", code, buf);
    return code;
}
#define CU(x)                                                                                         \
    do {                                                                                              \
        cudaError_t e_ = (x);                                                                         \
        if (e_ != cudaSuccess) return fail(DFFT_ECUDA, "%s:%d CUDA call '%s' failed: %s", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
    } while (0)

extern "C" const char* dfft_last_error(void) { return g_err.c_str(); }
extern "C" int dfft_version(void) { return 100; }

extern "C" int dfft_length_kind(int n, int precision)
{
    if (n < 1 || n > (1 << 20) || (precision != DFFT_DOUBLE && precision != DFFT_FLOAT)) return 0;
    const SizeEntry* e = find_size_entry(n, precision);
    return !e ? 0 : (e->gen ? 1 : 2);
}

/* radix schedule the library uses for length n (contiguous-pass schedule for tuned lengths, the run-time schedule for
 * generic ones); returns the number of stages, 0 if unsupported */
extern "C" int dfft_length_schedule(int n, int precision, int* radices, int max_radices)
{
    if (n < 1 || n > (1 << 20) || (precision != DFFT_DOUBLE && precision != DFFT_FLOAT)) return 0;
    const SizeEntry* e = find_size_entry(n, precision);
    if (!e) return 0;
    if (radices)
        for (int i = 0; i < e->z_nstages && i < max_radices; i++) radices[i] = e->z_rad[i];
    return e->z_nstages;
}

/* test hook (host only, no device needed): ticket -> (role, part, plane, tile) of the single-kernel forward path;
 * ticket < 0 returns the number of tickets */
extern "C" long long dfft_debug_fused3_order(long long planes, long long rows, int GA, int GBk, int GXk, int K, int lag, long long ticket, long long out[4])
{
    Fused3Ctl F{};
    F.planes = planes; F.rows = rows; F.GA = GA; F.GBk = GBk; F.GB = GBk * K; F.GXk = GXk; F.GX = GXk * K; F.K = K; F.lag = lag;
    const Fused3Order o = fused3_prepare(F);
    const long long total = (long long)o.total;
    if (ticket < 0 || ticket >= total || !out) return total;
    int role, part, yfloor;
    unsigned plane, idx;
    fused3_decode(F, o, (unsigned)ticket, role, part, plane, idx, yfloor);
    out[0] = role; out[1] = part; out[2] = plane; out[3] = idx;
    return total;
}

/* test hook (host only): ticket order of the two-role t0 kernels (fft_fused2_kernel, fft_tma_fused_zy_kernel); out = role
 * (0 first role, 1 second role), plane, tile; returns the number of tickets (ticket < 0: only that) */
extern "C" long long dfft_debug_fused2_order(long long planes, int GA, int GB, int lag, long long ticket, long long out[3])
{
    FusedCtl F{};
    F.planes = planes; F.GA = GA; F.GB = GB; F.lag = lag;
    const Fused2Order o = fused2_prepare(F);
    const long long total = (long long)o.total;
    if (ticket < 0 || ticket >= total || !out) return total;
    bool roleA;
    unsigned plane, idx;
    fused2_decode(o, (unsigned)ticket, roleA, plane, idx);
    out[0] = roleA ? 0 : 1; out[1] = plane; out[2] = idx;
    return total;
}

extern "C" int dfft_supported_lengths(int precision, int* lengths, int max_lengths)
{
    std::vector<int> v;
    list_sizes(precision, v);
    std::sort(v.begin(), v.end());
    if (lengths)
        for (int i = 0; i < (int)v.size() && i < max_lengths; i++) lengths[i] = v[i];
    return (int)v.size();
}

// ------------------------------------------------------------------------------------------------
// slab geometry (fft_mpi_3d_api.cpp:56-66, 89-91, 232-316)
// ------------------------------------------------------------------------------------------------
static inline long long cdiv(long long a, long long b) { return (a + b - 1) / b; }

struct Geom {
    long long n0, n1, n2;
    int P;
    long long xd() const { return cdiv(n0, P); }
    long long yd() const { return cdiv(n1, P); }
    long long last_n0() const { return n0 - (P - 1) * xd(); }
    long long last_n1() const { return n1 - (P - 1) * yd(); }
    long long n0l(int p) const { return p == P - 1 ? last_n0() : xd(); }
    long long n1l(int q) const { return q == P - 1 ? last_n1() : yd(); }
    long long in_count(int p) const { return n0l(p) * n1 * n2; }
    long long out_count(int q) const { return n0 * n1l(q) * n2; }
    long long max_count(int p) const { return std::max(in_count(p), out_count(p)); }
};

static int proper_device_num(long long n0, int wanted)
{
    if (wanted < 1) return 0;
    if (n0 % wanted == 0) return wanted;
    long long per = n0 / wanted + 1;
    int dev = (int)(n0 / per);
    if (n0 % per) dev += 1;
    return dev;
}

extern "C" int dfft_init(const long long N[3], int wanted, int* total, int* local, long long* counts)
{
    if (!N || wanted < 1 || N[0] < 1 || N[1] < 1 || N[2] < 1) return fail(DFFT_EINVAL, "dfft_init: bad arguments");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess) { cudaGetLastError(); ndev = 0; }
    if (ndev > 0 && wanted > ndev) wanted = ndev;   // api.cpp:236-239
    int dev = proper_device_num(N[0], wanted);
    if (dev < 1) return fail(DFFT_EUNSUPPORTED, "could not support this distribution of data");
    Geom g{N[0], N[1], N[2], dev};
    if (g.last_n1() < 1) return fail(DFFT_EUNSUPPORTED, "N1=%lld cannot be split over %d devices (empty last y-slab)", N[1], dev);
    if (counts)
        for (int i = 0; i < dev; i++) counts[i] = g.in_count(i);
    if (total) *total = dev;
    if (local) *local = dev;
    // peer access between the devices used (api.cpp:16-27)
    for (int i = 0; i < dev && i < ndev; i++) {
        int cur = 0;
        cudaGetDevice(&cur);
        if (cudaSetDevice(i) != cudaSuccess) { cudaGetLastError(); continue; }
        for (int j = 0; j < dev && j < ndev; j++) {
            if (i == j) continue;
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, i, j) == cudaSuccess && can) {
                cudaError_t pe = cudaDeviceEnablePeerAccess(j, 0);
                if (pe != cudaSuccess) cudaGetLastError();   // already enabled is fine
            }
        }
        cudaSetDevice(cur);
    }
    return 0;
}

extern "C" long long dfft_max_data_count(long long n0, long long n1, long long n2, int P, int is_last)
{
    if (P < 1) return -1;
    Geom g{n0, n1, n2, P};
    return g.max_count(is_last ? P - 1 : 0);
}

extern "C" long long dfft_local_size_3d(long long n0, long long n1, long long n2, int P, int dev, long long* ln0,
                                        long long* s0, long long* ln1, long long* s1)
{
    if (P < 1 || dev < 0 || dev >= P) return -1;
    Geom g{n0, n1, n2, P};
    if (ln0) *ln0 = g.n0l(dev);
    if (s0) *s0 = dev * g.xd();
    if (ln1) *ln1 = g.n1l(dev);
    if (s1) *s1 = dev * g.yd();
    return g.max_count(dev);
}

extern "C" void* dfft_alloc_local(long long count, int flag, int precision)
{
    if (count < 0) { fail(DFFT_EINVAL, "negative count"); return nullptr; }
    size_t bytes = (size_t)count * (precision == DFFT_FLOAT ? 8 : 16);
    if (bytes == 0) bytes = 16;
    void* p = nullptr;
    cudaError_t e;
    if (flag == DFFT_ALLOC_CPU) e = cudaMallocHost(&p, bytes);
    else if (flag == DFFT_ALLOC_DEV) e = cudaMalloc(&p, bytes);
    else { fail(DFFT_EINVAL, "Fail to allocate memory!"); return nullptr; }
    if (e != cudaSuccess) { fail(DFFT_ENOMEM, "allocation of %zu bytes failed: %s", bytes, cudaGetErrorString(e)); cudaGetLastError(); return nullptr; }
    return p;
}

extern "C" int dfft_free_local(void* p, int flag)
{
    if (!p) return 0;
    if (flag == DFFT_ALLOC_CPU) CU(cudaFreeHost(p));
    else CU(cudaFree(p));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// communicator
// ------------------------------------------------------------------------------------------------
struct dfft_comm_s {
    int nranks = 1;
    bool local = true;
    // local (threads of one process)
    std::mutex mu;
    std::condition_variable cv;
    int arrived = 0;
    long long gen = 0;
    std::vector<std::vector<unsigned char>> slots;
    // bootstrap (process per GPU)
    int rank = 0;
    dfft_allgather_fn ag = nullptr;
    void* ctx = nullptr;

    // A participant that fails in the middle of a collective sequence (plan creation) poisons the communicator: every
    // rank blocked in -- or later entering -- a barrier returns an error instead of waiting for a peer that will never come.
    bool failed = false;
    void poison()
    {
        std::lock_guard<std::mutex> lk(mu);
        failed = true;
        cv.notify_all();
    }
    int barrier()
    {
        std::unique_lock<std::mutex> lk(mu);
        if (failed) return -1;
        long long g = gen;
        if (++arrived == nranks) { arrived = 0; gen++; cv.notify_all(); }
        else cv.wait(lk, [&] { return gen != g || failed; });
        return failed ? -1 : 0;
    }
    int allgather(int r, const void* send, void* recv, size_t bytes)
    {
        if (nranks == 1) { memcpy(recv, send, bytes); return 0; }
        if (!local) return ag(ctx, send, recv, bytes);
        {
            std::lock_guard<std::mutex> lk(mu);
            slots[r].assign((const unsigned char*)send, (const unsigned char*)send + bytes);
        }
        if (barrier()) return -1;
        for (int i = 0; i < nranks; i++) memcpy((unsigned char*)recv + (size_t)i * bytes, slots[i].data(), bytes);
        if (barrier()) return -1;
        return 0;
    }
    int host_barrier(int r)
    {
        if (nranks == 1) return 0;
        if (local) return barrier();
        std::vector<unsigned char> tmp(nranks);
        unsigned char one = 1;
        return ag(ctx, &one, tmp.data(), 1);
    }
};

extern "C" int dfft_comm_create_local(int nranks, dfft_comm* comm)
{
    if (nranks < 1 || !comm) return fail(DFFT_EINVAL, "dfft_comm_create_local: bad arguments");
    dfft_comm c = new dfft_comm_s;
    c->nranks = nranks;
    c->local = true;
    c->slots.resize(nranks);
    *comm = c;
    return 0;
}

extern "C" int dfft_comm_create_bootstrap(int rank, int nranks, dfft_allgather_fn ag, void* ctx, dfft_comm* comm)
{
    if (nranks < 1 || rank < 0 || rank >= nranks || !comm || (nranks > 1 && !ag))
        return fail(DFFT_EINVAL, "dfft_comm_create_bootstrap: bad arguments");
    dfft_comm c = new dfft_comm_s;
    c->nranks = nranks;
    c->local = false;
    c->rank = rank;
    c->ag = ag;
    c->ctx = ctx;
    *comm = c;
    return 0;
}

/* host-side all-gather through the communicator (what plan creation uses to exchange IPC handles) */
extern "C" int dfft_comm_allgather(dfft_comm c, int rank, const void* send, void* recv, size_t bytes)
{
    if (!c || !send || !recv || rank < 0 || rank >= c->nranks) return fail(DFFT_EINVAL, "dfft_comm_allgather: bad arguments");
    if (c->allgather(rank, send, recv, bytes) != 0) return fail(DFFT_ECOMM, "bootstrap allgather failed");
    return 0;
}

extern "C" int dfft_comm_destroy(dfft_comm c)
{
    delete c;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// NCCL, loaded at run time (no link-time dependency; picks up the copy torch already loaded)
// ------------------------------------------------------------------------------------------------
struct NcclUid { char b[128]; };   // ncclUniqueId (NCCL_UNIQUE_ID_BYTES = 128), passed by value
struct NcclApi {
    void* h = nullptr;
    int (*GetUniqueId)(NcclUid*) = nullptr;
    int (*CommInitRank)(void**, int, NcclUid, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*AlltoAll)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;   // NCCL >= 2.28
    const char* (*GetErrorString)(int) = nullptr;
    int (*GetVersion)(int*) = nullptr;
    bool ok = false;
};

static NcclApi& nccl_api()
{
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* names[] = {getenv("DFFT_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            if (!n) continue;
            api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.h) break;
        }
        if (!api.h) return;
#define LD(field, sym) *(void**)(&api.field) = dlsym(api.h, sym)
        LD(GetUniqueId, "ncclGetUniqueId");
        LD(CommInitRank, "ncclCommInitRank");
        LD(CommDestroy, "ncclCommDestroy");
        LD(GroupStart, "ncclGroupStart");
        LD(GroupEnd, "ncclGroupEnd");
        LD(Send, "ncclSend");
        LD(Recv, "ncclRecv");
        LD(AlltoAll, "ncclAlltoAll");
        LD(GetErrorString, "ncclGetErrorString");
        LD(GetVersion, "ncclGetVersion");
#undef LD
        api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.GroupStart && api.GroupEnd && api.Send && api.Recv;
    });
    return api;
}
#define NC(x)                                                                                          \
    do {                                                                                               \
        int r_ = (x);                                                                                  \
        if (r_ != 0) return fail(DFFT_ECOMM, "%s:%d NCCL call '%s' failed: %s", __FILE__, __LINE__, #x, \
                                 nccl_api().GetErrorString ? nccl_api().GetErrorString(r_) : "?");     \
    } while (0)

// ------------------------------------------------------------------------------------------------
// cross-device flags for the fused (P2P) exchange
// ------------------------------------------------------------------------------------------------
struct SyncBlock {
    unsigned long long arrive[DFFT_MAX_CHUNKS];  // arrive[s] = e : sender s finished writing my recv buffer for epoch e
    unsigned long long ready[DFFT_MAX_CHUNKS];   // ready[r] = e  : receiver r finished reading its recv buffer of epoch e
    unsigned long long part_arrive[DFFT_MAX_PARTS][DFFT_MAX_CHUNKS];   // overlapped mode: part k of sender s has arrived (epoch e)
};
struct FlagPtrs {
    unsigned long long* p[DFFT_MAX_CHUNKS];
};

__global__ void signal_flags_kernel(FlagPtrs dst, int n, unsigned long long value)
{
    const int q = threadIdx.x;
    if (q < n) {
        __threadfence_system();
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(dst.p[q]), "l"(value) : "memory");
    }
}
__global__ void wait_flags_kernel(const unsigned long long* flags, int n, unsigned long long value)
{
    const int q = threadIdx.x;
    if (q < n) {
        unsigned long long v;
        SpinGuard guard;   // a peer that never signals (it died) traps this kernel after DFFT_SPIN_TIMEOUT_NS instead of hanging the GPU
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flags + q) : "memory");
            if (v < value) { __nanosleep(200); guard.tick(); }
        } while (v < value);
    }
    __threadfence_system();
}

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
struct dfft_plan_s {
    Geom g;
    int P = 1, me = 0, direction = DFFT_FORWARD, prec = 0, device = 0, sms = 132;
    unsigned flags = 0;
    int xmode = DFFT_EXCHANGE_P2P;
    size_t esz = 16;
    long long n0l = 0, n1l = 0, in_count = 0, out_count = 0, max_count = 0;
    void *in = nullptr, *out = nullptr, *buf1 = nullptr, *buf2 = nullptr;
    void* work = nullptr;   // plan-owned scratch / receive buffer: keeps bufferDev1 intact so execute is repeatable
    bool inplace = false;
    const SizeEntry *ez = nullptr, *ey = nullptr, *ex = nullptr;   // axes N2 (Z), N1 (Y), N0 (X)
    void *lut_z = nullptr, *lut_y = nullptr, *lut_x = nullptr;
    void* lut_xn = nullptr;   // X axis with the strided-local schedule (DFFT_NATURAL_SPECTRUM)
    // TMA-pipelined pass kernels (fft_tma.cuh) for the axes that have an instantiation: used for the passes whose load and
    // store are both local and un-chunked (Z, natural Y, X with the fused transpose); nullptr -> register-staged kernels
    const TmaEntry *tz = nullptr, *ty = nullptr, *tx = nullptr;
    void *lut_tz = nullptr, *lut_ty = nullptr, *lut_tx = nullptr;
    bool natural = false;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t pev[3][2] = {{nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}};   // per pass (Z, Y, X) brackets
    dfft_comm comm = nullptr;
    // p2p
    std::vector<void*> peer_work, peer_buf1;
    SyncBlock* sync = nullptr;
    std::vector<SyncBlock*> peer_sync;
    std::vector<void*> ipc_opened;
    unsigned long long epoch = 0;
    // nccl
    void* nccl = nullptr;
    int launches = 0;
    bool timed = false;
    // fused two-pass t0 (L2-resident intermediate): per-plane completion counters + ticket words
    bool fuse = false;
    bool fuse_tma = false;   // forward, one device: t0 runs on the TMA fused kernel of tz (fft_tma_fused_zy_kernel)
    int lag = 0;
    unsigned long long* plane_done = nullptr;
    unsigned int* ticket = nullptr;
    unsigned long long fuse_epoch = 0;   // plane_done value every plane reaches once the last fused launch is done (sum of its GA)
    // describe-only plans (DFFT_DRY_RUN): no CUDA call is made, buffers are symbolic addresses, execute records the
    // passes it would launch (dfft_debug_plan_ops) -- lets the CPU tests interpret the whole multi-device schedule
    bool dry = false;
    std::vector<std::string> ops;
    // overlapped forward (fft_fused3_kernel): own intermediate buffer, per-part counters
    bool overlap = false;
    int parts = 1;
    void* mid = nullptr;
    unsigned long long* part_done = nullptr;
    unsigned long long overlap_epoch = 0;
    // stream-pipelined forward (DFFT_PIPELINE): the z axis is cut into `parts`; the send side (stream: Z, then the Y pass of
    // part k with the pack / peer stores folded in, or + ncclAlltoAll of part k on the comm stream) runs ahead of the receive
    // side (stream2: X pass of part k as soon as part k has arrived from every sender) -- t2 and t3 overlap t0
    bool pipe = false;
    bool pipe_fyx = false;           // forward, cube, P2P: parts run as a chain of two-role kernels on ONE stream (fft_fused_yx_kernel:
                                     // Y pass of part k + X pass of part k-1 share every SM slot) instead of two streams
    bool in_pipe = false;            // inside fwd_pipelined: Pass::launch leaves the per-pass event brackets alone
    cudaStream_t stream2 = nullptr, stream3 = nullptr;   // receive side; NCCL part exchanges
    cudaEvent_t ev_join = nullptr, evb[2] = {nullptr, nullptr};
    cudaEvent_t ev_y[DFFT_MAX_PARTS] = {}, ev_a[DFFT_MAX_PARTS] = {};
    void* sendbuf = nullptr;         // NCCL: part-major packed send buffer
    unsigned long long* dbg = nullptr;   // DFFT_DEBUG_TIMELINE: device-side timeline of the single-kernel forward path
    unsigned int* done_ctr = nullptr; // [DFFT_MAX_PARTS] finished-CTA counters of the part kernels (arrival signal folded into the kernel)
    // real-data plans (dfft_plan_r2c_3d): g.n2 is the half-spectrum extent nzh = n2r / 2 + 1, which is all the Y, X and exchange
    // code sees; only the Z pass (fft_real.cuh) and the scale factor use the real length n2r.  in_count / out_count are in
    // elements of each side's own type (in_esz / out_esz bytes)
    bool r2c = false;
    long long n2r = 0;
    size_t in_esz = 16, out_esz = 16;
    // spectral convolution plans (dfft_plan_convolve_*): forward half, fused X pass (forward x, multiply, inverse x), backward half,
    // each half run with its own direction and fused choice (`direction` stays DFFT_FORWARD)
    bool conv = false;
    bool conv_fuse[2] = {false, false};   // fused t0 of the forward [0] / backward [1] half, chosen as a C2C plan of that direction would
    bool conv_fuse_tma = false;           // the forward half's t0 is the TMA fused kernel
    void* work2 = nullptr;                // P2P convolve: the backward exchange's receive buffer (the peers store into it while this
    std::vector<void*> peer_work2;        // device may still be reading `work`)
    // buffer roles of the slab schedule (execute_slabs): `stage` = the P2P forward Z output and the NCCL send buffer of either
    // direction, `ybwd` = the backward Y output.  C2C plans borrow bufferDev2; R2C and convolve plans use `mid`, so that a user's
    // real buffer never holds complex data (a one-device R2C plan runs its backward Y in place in `work`)
    void* stage = nullptr;
    void* ybwd = nullptr;
};

// symbolic device address of a describe-only plan: device d (0-based), buffer id b: 1 bufferDev1, 2 bufferDev2 / user out,
// 3 work / receive buffer, 4 intermediate of the single-kernel path, 5 user in
static inline void* fake_addr(int d, int b) { return (void*)((((unsigned long long)(d + 1)) << 44) | (((unsigned long long)b) << 40)); }
static inline char* eoff(void* base, long long elems, size_t esz) { return (char*)base + (size_t)elems * esz; }
static inline cudaError_t ev_record(dfft_plan p, cudaEvent_t e) { return p->dry ? cudaSuccess : cudaEventRecord(e, p->stream); }
static inline cudaError_t ev_record_on(dfft_plan p, cudaEvent_t e, cudaStream_t st) { return p->dry ? cudaSuccess : cudaEventRecord(e, st); }
static inline cudaError_t stream_wait(dfft_plan p, cudaStream_t st, cudaEvent_t e) { return p->dry ? cudaSuccess : cudaStreamWaitEvent(st, e, 0); }

static const char* const kPassNames[PK_COUNT] = {"Z", "Y", "Y_CO", "Y_CI", "XF", "XB", "XB_CO", "XF_TW", "Z_R2C", "Z_C2R", "XCONV", "XCONV_CO",
                                                  "XY_PLANE", "XY_PLANE_CONV", "LINE_CONV", "LINE_CONV_R2C"};

// `extra`: further fields of the record, each starting with ", "
template <typename T>
static void record_op(std::vector<std::string>& ops, const char* name, int phase, int N, int C, bool chunk_in, bool chunk_out, bool transposed_store,
                      const TileArgs<T>& a, const char* extra = "")
{
    char buf[256];
    std::string o = "{";
    snprintf(buf, sizeof(buf), "\"op\": \"%s\", \"phase\": %d, \"N\": %d, \"C\": %d, \"G\": %d, \"W\": %d, \"ntiles\": %lld, \"inv\": %d, \"do_scale\": %d, \"scale\": %.17g, \"tw_n\": %lld, ",
             name, phase, N, C, a.G, a.W, a.ntiles, a.inv, a.do_scale, (double)a.scale, a.tw_n);
    o += buf;
    snprintf(buf, sizeof(buf), "\"in\": %llu, \"out\": %llu, \"ia\": [%lld, %lld, %lld, %lld], \"oa\": [%lld, %lld, %lld, %lld], \"tstore\": %d",
             (unsigned long long)(size_t)a.in, (unsigned long long)(size_t)a.out, a.ia.SA, a.ia.SB, a.ia.cs, a.ia.es, a.oa.SA, a.oa.SB, a.oa.cs, a.oa.es,
             transposed_store ? 1 : 0);
    o += buf;
    for (int side = 0; side < 2; side++) {
        const bool on = side == 0 ? chunk_in : chunk_out;
        if (!on) continue;
        const ChunkTab& ct = side == 0 ? a.ci : a.co;
        snprintf(buf, sizeof(buf), ", \"%s\": {\"ediv\": %d, \"nchunks\": %d, \"cptr\": [", side == 0 ? "ci" : "co", ct.ediv, ct.nchunks);
        o += buf;
        for (int q = 0; q < ct.nchunks; q++) { snprintf(buf, sizeof(buf), "%s%llu", q ? ", " : "", (unsigned long long)(size_t)ct.cptr[q]); o += buf; }
        o += "], \"SAq\": [";
        for (int q = 0; q < ct.nchunks; q++) { snprintf(buf, sizeof(buf), "%s%lld", q ? ", " : "", ct.SAq[q]); o += buf; }
        o += "]}";
    }
    o += extra;
    o += "}";
    ops.push_back(o);
}

// the records as one JSON array (the debug hooks' format); returns the bytes needed, copied into buf when cap suffices
static long long ops_json(const std::vector<std::string>& ops, char* buf, long long cap)
{
    std::string o = "[";
    for (size_t i = 0; i < ops.size(); i++) { if (i) o += ", "; o += ops[i]; }
    o += "]";
    if (buf && cap > (long long)o.size()) memcpy(buf, o.c_str(), o.size() + 1);
    return (long long)o.size() + 1;
}

template <typename T> static cudaError_t upload_lut(void** dst, int nstages, const int* rad)
{
    std::vector<cx<T>> lut = build_lut<T>(nstages, rad);
    cudaError_t e = cudaMalloc(dst, lut.size() * sizeof(cx<T>));
    if (e != cudaSuccess) { *dst = nullptr; return e; }
    return cudaMemcpy(*dst, lut.data(), lut.size() * sizeof(cx<T>), cudaMemcpyHostToDevice);
}

// lines per tile of a pass kind's kernel in entry e: contiguous (Z), strided local (Y, unpack load, convolution X pass), peer /
// packed store (Y with the chunked store, chunked convolution X pass), X passes
static int kind_C(const SizeEntry* e, int kind)
{
    switch (kind) {
    case PK_Z: return e->z_C;
    case PK_Y: case PK_XCONV: return e->s_C;
    case PK_Y_CI: return e->ci_C;
    case PK_Y_CO: case PK_XCONV_CO: return e->p_C;
    case PK_XB_CO: return e->xo_C;
    default: return e->x_C;
    }
}

// twiddle table of the radix schedule a pass kind's kernel runs: the contiguous one (Z), the X one (forward / backward X passes),
// the strided one otherwise (Y kinds; the convolution X pass, as the natural-order X pass)
template <typename T> static cudaError_t upload_lut_kind(void** dst, const SizeEntry* e, int kind)
{
    if (kind == PK_Z) return upload_lut<T>(dst, e->z_nstages, e->z_rad);
    if (kind == PK_XF || kind == PK_XB || kind == PK_XB_CO || kind == PK_XF_TW) return upload_lut<T>(dst, e->x_nstages, e->x_rad);
    return upload_lut<T>(dst, e->s_nstages, e->s_rad);
}

static int share_pointer(dfft_plan p, void* mine, std::vector<void*>& peers)
{
    // make `mine` (a cudaMalloc allocation of this device) addressable by every rank
    const int P = p->P;
    peers.assign(P, nullptr);
    if (p->dry) return 0;   // describe-only plans compute peer addresses symbolically
    if (p->comm->local) {
        std::vector<void*> all(P);
        if (p->comm->allgather(p->me, &mine, all.data(), sizeof(void*)) != 0) return fail(DFFT_ECOMM, "a peer failed during plan creation");
        peers = all;
        return 0;
    }
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, mine));
    std::vector<cudaIpcMemHandle_t> all(P);
    if (p->comm->allgather(p->me, &h, all.data(), sizeof(h)) != 0) return fail(DFFT_ECOMM, "bootstrap allgather failed");
    for (int q = 0; q < P; q++) {
        if (q == p->me) { peers[q] = mine; continue; }
        void* ptr = nullptr;
        CU(cudaIpcOpenMemHandle(&ptr, all[q], cudaIpcMemLazyEnablePeerAccess));
        peers[q] = ptr;
        p->ipc_opened.push_back(ptr);
    }
    return 0;
}

static int plan_create(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                       int P, int direction, int precision, unsigned flags, dfft_plan* plan_out, bool real, bool conv);

// a participant that fails (bad argument, allocation, peer mapping ...) must not leave the others waiting for it in the collective
// part of plan creation: the local communicator is poisoned and their barriers return an error
static int plan_create_collective(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx, int P,
                                  int direction, int precision, unsigned flags, dfft_plan* plan_out, bool real, bool conv)
{
    const int rc = plan_create(n0, n1, n2, in, out, comm, dev_idx, P, direction, precision, flags, plan_out, real, conv);
    if (rc != 0 && P > 1 && comm && comm->local && !(flags & DFFT_DRY_RUN)) comm->poison();
    return rc;
}

extern "C" int dfft_plan_c2c_3d(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                                int P, int direction, int precision, unsigned flags, dfft_plan* plan_out)
{
    return plan_create_collective(n0, n1, n2, in, out, comm, dev_idx, P, direction, precision, flags, plan_out, false, false);
}

extern "C" int dfft_plan_r2c_3d(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                                int P, int direction, int precision, unsigned flags, dfft_plan* plan_out)
{
    return plan_create_collective(n0, n1, n2, in, out, comm, dev_idx, P, direction, precision, flags, plan_out, true, false);
}

extern "C" int dfft_plan_convolve_c2c_3d(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                                         int P, int precision, unsigned flags, dfft_plan* plan_out)
{
    return plan_create_collective(n0, n1, n2, in, out, comm, dev_idx, P, DFFT_FORWARD, precision, flags, plan_out, false, true);
}

extern "C" int dfft_plan_convolve_r2c_3d(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                                         int P, int precision, unsigned flags, dfft_plan* plan_out)
{
    return plan_create_collective(n0, n1, n2, in, out, comm, dev_idx, P, DFFT_FORWARD, precision, flags, plan_out, true, true);
}

extern "C" int dfft_local_size_r2c_3d(long long n0, long long n1, long long n2, int P, int dev, long long* real_count, long long* complex_count)
{
    if (P < 1 || dev < 0 || dev >= P || n0 < 1 || n1 < 1 || n2 < 1) return fail(DFFT_EINVAL, "dfft_local_size_r2c_3d: bad arguments");
    Geom g{n0, n1, n2 / 2 + 1, P};
    if (g.last_n0() < 1 || g.last_n1() < 1) return fail(DFFT_EUNSUPPORTED, "%lldx%lldx%lld cannot be split over %d devices (empty last slab)", n0, n1, n2, P);
    if (real_count) *real_count = g.n0l(dev) * n1 * n2;
    if (complex_count) *complex_count = g.out_count(dev);
    return 0;
}

static int plan_create(long long n0, long long n1, long long n2, void* in, void* out, dfft_comm comm, int dev_idx,
                       int P, int direction, int precision, unsigned flags, dfft_plan* plan_out, bool real, bool conv)
{
    const char* what = conv ? (real ? "dfft_plan_convolve_r2c_3d" : "dfft_plan_convolve_c2c_3d") : (real ? "dfft_plan_r2c_3d" : "dfft_plan_c2c_3d");
    if (!plan_out) return fail(DFFT_EINVAL, "null plan pointer");
    *plan_out = nullptr;
    if (n0 < 1 || n1 < 1 || n2 < 1 || P < 1 || dev_idx < 0 || dev_idx >= P || !in)
        return fail(DFFT_EINVAL, "%s: bad arguments", what);
    if (direction != DFFT_FORWARD && direction != DFFT_BACKWARD) return fail(DFFT_EINVAL, "direction must be +1 or -1");
    if (precision != DFFT_DOUBLE && precision != DFFT_FLOAT) return fail(DFFT_EINVAL, "bad precision");
    if (P > DFFT_MAX_CHUNKS) return fail(DFFT_EUNSUPPORTED, "at most %d devices", DFFT_MAX_CHUNKS);
    const bool dry = (flags & DFFT_DRY_RUN) != 0;
    if (conv) {
        // a convolve plan exposes no spectrum, and its two exchanges are folded into its kernels or handed to NCCL
        if (flags & DFFT_NATURAL_SPECTRUM) return fail(DFFT_EINVAL, "%s: DFFT_NATURAL_SPECTRUM has no meaning for a convolve plan (no spectrum is exposed)", what);
        if ((flags & DFFT_EXCHANGE_MASK) == DFFT_EXCHANGE_STAGED) return fail(DFFT_EUNSUPPORTED, "%s: DFFT_EXCHANGE_STAGED is not supported", what);
    } else if (real) {
        // the real and the complex slab differ in size and layout: no in-place (padded) layout, no stage-by-stage mode
        if (!out || out == in) return fail(DFFT_EINVAL, "dfft_plan_r2c_3d: `out` must be a separate buffer (in-place R2C is not supported)");
        if ((flags & DFFT_EXCHANGE_MASK) == DFFT_EXCHANGE_STAGED) return fail(DFFT_EUNSUPPORTED, "R2C / C2R plans do not support DFFT_EXCHANGE_STAGED");
    }
    if (!dry && P > 1 && (!comm || comm->nranks != P)) return fail(DFFT_EINVAL, "a communicator of %d ranks is required", P);
    Geom g{n0, n1, real ? n2 / 2 + 1 : n2, P};   // R2C: everything but the Z pass works on the nzh = n2/2 + 1 half-spectrum columns
    if (g.last_n0() < 1 || g.last_n1() < 1)
        return fail(DFFT_EUNSUPPORTED, "%lldx%lldx%lld cannot be split over %d devices (empty last slab); use dfft_init", n0, n1, n2, P);
    const SizeEntry* ez = find_size_entry((int)n2, precision);
    const SizeEntry* ey = find_size_entry((int)n1, precision);
    const SizeEntry* ex = find_size_entry((int)n0, precision);
    if (n0 > 1 << 20 || n1 > 1 << 20 || n2 > 1 << 20 || !ez || !ey || !ex)
        return fail(DFFT_EUNSUPPORTED, "unsupported transform length in %lldx%lldx%lld (see dfft_supported_lengths)", n0, n1, n2);
    if (real && (ez->gen || !ez->launch[PK_Z_R2C] || !ez->launch[PK_Z_C2R]))
        return fail(DFFT_EUNSUPPORTED, "R2C / C2R needs a z length with a tuned kernel (dfft_length_kind == 2); %lld has none", n2);
    if (conv && (ex->gen || !ex->launch[PK_XCONV] || !ex->launch[PK_XCONV_CO]))
        return fail(DFFT_EUNSUPPORTED, "%s: the x length %lld has no convolution kernel (it needs a tuned length, dfft_length_kind == 2, of the default kernel table)", what, n0);
    // bufferDev2 (`out`, or `in` in place) is written by the pass kernels; an out-of-place `in` is only copied (cudaMemcpy).
    // TMA needs 16-byte-aligned global addresses, and so do the fp64 kernels' double2 accesses: such a buffer is rejected in
    // fp64, and in fp32 (float2 accesses, 8 bytes) it keeps the plan on the register-staged kernels.  R2C plans apply the rule
    // to their complex-side buffer (forward `out`, backward `in`); the real side only needs the alignment of its element type
    // A real convolve plan keeps every complex array in plan-owned buffers: its user buffers only need their element alignment
    const void* cbuf = real ? (direction == DFFT_FORWARD ? out : in) : ((!out || out == in) ? in : out);
    const bool buf2_aligned = (real && conv) || ((uintptr_t)cbuf & 15) == 0;
    if (precision == DFFT_DOUBLE && !buf2_aligned) return fail(DFFT_EINVAL, "a double-precision output buffer must be 16-byte aligned");
    const size_t rsz = precision == DFFT_FLOAT ? 4 : 8;
    if (real && !conv && ((uintptr_t)(direction == DFFT_FORWARD ? in : out) % rsz) != 0) return fail(DFFT_EINVAL, "the real buffer is not aligned to its element size");
    if (real && conv && (((uintptr_t)in % rsz) != 0 || (out && ((uintptr_t)out % rsz) != 0))) return fail(DFFT_EINVAL, "the real buffers are not aligned to their element size");

    dfft_plan p = new dfft_plan_s;
    p->g = g; p->P = P; p->me = dev_idx; p->direction = direction; p->prec = precision; p->flags = flags;
    p->esz = precision == DFFT_FLOAT ? 8 : 16;
    p->n0l = g.n0l(dev_idx); p->n1l = g.n1l(dev_idx);
    p->in_count = direction == DFFT_FORWARD ? g.in_count(dev_idx) : g.out_count(dev_idx);
    p->out_count = direction == DFFT_FORWARD ? g.out_count(dev_idx) : g.in_count(dev_idx);
    p->max_count = g.max_count(dev_idx);
    p->in_esz = p->out_esz = p->esz;
    if (real) {
        p->r2c = true;
        p->n2r = n2;
        const long long rcount = p->n0l * n1 * n2;
        if (direction == DFFT_FORWARD) { p->in_count = rcount; p->in_esz = rsz; }
        else { p->out_count = rcount; p->out_esz = rsz; }
    }
    if (conv) {
        // input and output are both exactly this device's x-slab
        p->conv = true;
        p->in_count = p->out_count = p->n0l * n1 * n2;
        p->in_esz = p->out_esz = real ? rsz : p->esz;
    }
    p->ez = ez; p->ey = ey; p->ex = ex; p->comm = comm;
    p->in = in; p->out = out;
    p->dry = dry;
    int rc = 0;
    // a rank that fails after the collective part has begun must not leave its peers waiting for it
    auto bail = [&](int code) { if (!dry && P > 1 && comm && comm->local) comm->poison(); dfft_destroy(p); return code; };   // poison BEFORE destroy's barrier
#define CUP(x)                                                                                        \
    do {                                                                                              \
        cudaError_t e_ = (x);                                                                         \
        if (e_ != cudaSuccess) return bail(fail(DFFT_ECUDA, "%s:%d CUDA call '%s' failed: %s", __FILE__, __LINE__, #x, cudaGetErrorString(e_))); \
    } while (0)
    if (!dry) {
        CUP(cudaGetDevice(&p->device));
        CUP(cudaDeviceGetAttribute(&p->sms, cudaDevAttrMultiProcessorCount, p->device));
    }
    // buffers (api.cpp:66-77)
    if (!out || out == in) { p->inplace = true; p->buf2 = in; }
    else p->buf2 = out;
    if (dry) p->buf1 = fake_addr(dev_idx, 1);
    else {
        // R2C: bufferDev1 holds exactly the input slab (the user's buffer has only that many elements of its type)
        // convolve plans: the user's buffers are exactly the x-slab as well
        const size_t b1 = (p->r2c || conv) ? (size_t)p->in_count * p->in_esz : (size_t)p->max_count * p->esz;
        CUP(cudaMalloc(&p->buf1, b1));
        CUP(cudaMemcpy(p->buf1, in, b1, cudaMemcpyDeviceToDevice));
        CUP(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
        for (auto& e : p->ev) CUP(cudaEventCreate(&e));
        for (auto& pe : p->pev) for (auto& e : pe) CUP(cudaEventCreate(&e));
    }
    if (dry) {
        // no twiddle tables: the interpreter of the recorded passes does its own transforms
    } else if (precision == DFFT_DOUBLE) {
        CUP(upload_lut_kind<double>(&p->lut_z, ez, PK_Z));
        CUP(upload_lut_kind<double>(&p->lut_y, ey, PK_Y));
        CUP(upload_lut_kind<double>(&p->lut_x, ex, PK_XF));
    } else {
        CUP(upload_lut_kind<float>(&p->lut_z, ez, PK_Z));
        CUP(upload_lut_kind<float>(&p->lut_y, ey, PK_Y));
        CUP(upload_lut_kind<float>(&p->lut_x, ex, PK_XF));
    }
    if (conv && !dry) {   // the fused X pass runs the x entry's strided schedule (as the natural-order X pass does)
        if (precision == DFFT_DOUBLE) CUP(upload_lut_kind<double>(&p->lut_xn, ex, PK_XCONV));
        else CUP(upload_lut_kind<float>(&p->lut_xn, ex, PK_XCONV));
    }
    if (!dry) CUP(cudaGetLastError());
    if (!dry && !(flags & DFFT_NO_TMA) && buf2_aligned) {
        p->tz = real ? nullptr : find_tma_entry((int)n2, precision);   // R2C: the Z pass is always the real-data kernel
        p->ty = find_tma_entry((int)n1, precision);
        p->tx = find_tma_entry((int)n0, precision);
        const TmaEntry* te[3] = {p->tz, p->ty, p->tx};
        void** tl[3] = {&p->lut_tz, &p->lut_ty, &p->lut_tx};
        for (int i = 0; i < 3; i++) {
            if (!te[i]) continue;
            if (precision == DFFT_DOUBLE) CUP(upload_lut<double>(tl[i], te[i]->nstages, te[i]->rad));
            else CUP(upload_lut<float>(tl[i], te[i]->nstages, te[i]->rad));
        }
    }
    if (flags & DFFT_NATURAL_SPECTRUM) {
        // spectrum kept in natural [x][y][z] order: one device only (with P > 1 it would need a second all-to-all)
        if (P != 1) return bail(fail(DFFT_EUNSUPPORTED, "DFFT_NATURAL_SPECTRUM needs a single device (a distributed natural-order spectrum would take a second exchange)"));
        if ((flags & DFFT_EXCHANGE_MASK) == DFFT_EXCHANGE_STAGED) return bail(fail(DFFT_EINVAL, "DFFT_NATURAL_SPECTRUM cannot be combined with the staged mode"));
        p->natural = true;
        if (!dry) {
            if (precision == DFFT_DOUBLE) CUP(upload_lut<double>(&p->lut_xn, ex->s_nstages, ex->s_rad));
            else CUP(upload_lut<float>(&p->lut_xn, ex->s_nstages, ex->s_rad));
        }
    }
    // exchange mode
    int xmode = (int)(flags & DFFT_EXCHANGE_MASK);
    if (P == 1) xmode = xmode == DFFT_EXCHANGE_STAGED ? DFFT_EXCHANGE_STAGED : DFFT_EXCHANGE_P2P;
    else if (xmode == DFFT_EXCHANGE_AUTO) {
        const char* env = getenv("DFFT_EXCHANGE");
        if (env && !strcmp(env, "nccl")) xmode = DFFT_EXCHANGE_NCCL;
        else if (env && !strcmp(env, "staged")) xmode = DFFT_EXCHANGE_STAGED;
        else xmode = DFFT_EXCHANGE_P2P;
    }
    if (P > 1 && !dry) {
        // peer reachability (api.cpp:16-27 enables peer access in fft_mpi_init; done here so a plan does not
        // depend on dfft_init having run).  Threads of one process map peers directly and need
        // cudaDeviceEnablePeerAccess; separate processes get it from cudaIpcOpenMemHandle.
        std::vector<int> devs(P);
        if (comm->allgather(p->me, &p->device, devs.data(), sizeof(int)) != 0) return bail(fail(DFFT_ECOMM, "bootstrap allgather failed"));
        int reach = 1;
        if (comm->local) {
            for (int q = 0; q < P; q++) {
                if (q == p->me || devs[q] == p->device) continue;
                int can = 0;
                if (cudaDeviceCanAccessPeer(&can, p->device, devs[q]) != cudaSuccess || !can) { cudaGetLastError(); reach = 0; continue; }
                cudaError_t pe = cudaDeviceEnablePeerAccess(devs[q], 0);
                if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) reach = 0;
                cudaGetLastError();
            }
        }
        std::vector<int> all(P);
        if (comm->allgather(p->me, &reach, all.data(), sizeof(int)) != 0) return bail(fail(DFFT_ECOMM, "bootstrap allgather failed"));
        for (int q = 0; q < P; q++) reach &= all[q];
        if (!reach) {
            if ((flags & DFFT_EXCHANGE_MASK) == DFFT_EXCHANGE_AUTO && !getenv("DFFT_EXCHANGE")) xmode = DFFT_EXCHANGE_NCCL;
            else if (xmode != DFFT_EXCHANGE_NCCL) return bail(fail(DFFT_ECOMM, "peer access between the devices is not available; use DFFT_EXCHANGE_NCCL"));
        }
    }
    p->xmode = xmode;
    if (real && xmode == DFFT_EXCHANGE_STAGED) return bail(fail(DFFT_EUNSUPPORTED, "R2C / C2R plans do not support the staged exchange (DFFT_EXCHANGE=staged)"));
    // the fused kernels pair the contiguous and the strided role of one table entry: square planes only
    {
        // policy: the fused kernel wins when the strided role's stores are NVLink-bound (P2P exchange: the
        // contiguous role then hides entirely under the link time).  On one device the register-staged fused kernel
        // loses to the TMA-pipelined sweeps, but the TMA fused kernel (fft_tma_fused_zy_kernel) beats them where it is
        // instantiated and measured (TmaEntry::use bit TMA_USE_ZY, DESIGN.md 3.4): it is the default forward t0 there.
        // Forced fusion takes the TMA kernel whenever one exists, the register-staged kernel otherwise.
        const char* env = getenv("DFFT_FUSE");
        // t0 of one direction; a convolve plan selects each of its halves as the C2C plan of that direction would
        auto pick = [&](int dir, bool& fuse, bool& fuse_tma) {
            const bool tma_zy = P == 1 && dir == DFFT_FORWARD && n1 == n2 && !dry && p->tz && p->tz->fused_zy != nullptr && n2 % p->tz->C == 0;
            // the register-staged kind this plan would launch (zy_fused, and the part kernels of the pipelined schedules) must exist:
            // an entry leaves a kind null when its roles do not fit in shared memory together
            const int kind = dir == DFFT_FORWARD ? (P == 1 ? FK_ZY : FK_ZY_CO) : (P == 1 ? FK_YZ : FK_YZ_CI);
            const bool can = n1 == n2 && (ez->fused[kind] != nullptr || tma_zy);
            bool want = (P > 1 && xmode == DFFT_EXCHANGE_P2P) || (tma_zy && (p->tz->use & (1u << TMA_USE_ZY)));
            if (env) want = strcmp(env, "0") != 0;
            if (flags & DFFT_FORCE_FUSE) want = true;
            if (flags & DFFT_NO_FUSE) want = false;
            fuse = can && want && !real;   // R2C: the real Z pass has no fused form; the fusion flags are accepted and do nothing
            fuse_tma = fuse && tma_zy;
        };
        if (conv) {
            bool unused = false;
            pick(DFFT_FORWARD, p->conv_fuse[0], p->conv_fuse_tma);
            pick(DFFT_BACKWARD, p->conv_fuse[1], unused);
            p->fuse = p->conv_fuse[0] || p->conv_fuse[1];   // the plan holds the state a fused t0 of either half needs
        } else {
            pick(direction, p->fuse, p->fuse_tma);
        }
        if (getenv("DFFT_LAG")) p->lag = atoi(getenv("DFFT_LAG"));
        if (p->fuse && !dry) {
            CUP(cudaMalloc((void**)&p->plane_done, (size_t)p->n0l * sizeof(unsigned long long)));
            CUP(cudaMemset(p->plane_done, 0, (size_t)p->n0l * sizeof(unsigned long long)));
            CUP(cudaMalloc((void**)&p->ticket, 4 * sizeof(unsigned int)));
            CUP(cudaMemset(p->ticket, 0, 4 * sizeof(unsigned int)));
        }
    }

    if (dry && xmode == DFFT_EXCHANGE_STAGED) return bail(fail(DFFT_EINVAL, "DFFT_DRY_RUN cannot describe the staged mode"));
    if (dry) p->work = fake_addr(dev_idx, 3);
    else if (xmode != DFFT_EXCHANGE_STAGED) CUP(cudaMalloc(&p->work, (size_t)p->max_count * p->esz));
    {
        // opt-in: the whole forward transform of a device as one kernel with t3 overlapped behind per-part arrivals
        const char* env = getenv("DFFT_OVERLAP");
        const bool want = (flags & DFFT_OVERLAP_X) || (env && strcmp(env, "0") != 0);
        if (want && !conv && P > 1 && xmode == DFFT_EXCHANGE_P2P && direction == DFFT_FORWARD && p->fuse && ez->fused3 && ex == ez) {
            const int cy = ez->p_C, cx_ = ez->x_C;
            int lcm = cy > cx_ ? cy : cx_;   // both are powers of two in the tuned tables
            if (lcm % cy == 0 && lcm % cx_ == 0) {
                int K = 1;
                for (int k : {4, 2})
                    if (n2 % ((long long)k * lcm) == 0) { K = k; break; }
                if (getenv("DFFT_PARTS")) {
                    const int k = atoi(getenv("DFFT_PARTS"));
                    if (k >= 1 && k <= DFFT_MAX_PARTS && n2 % ((long long)k * lcm) == 0) K = k;
                }
                p->parts = K;
                p->overlap = true;
                if (dry) p->mid = fake_addr(dev_idx, 4);
                else {
                    CUP(cudaMalloc(&p->mid, (size_t)p->max_count * p->esz));
                    CUP(cudaMalloc((void**)&p->part_done, DFFT_MAX_PARTS * sizeof(unsigned long long)));
                    CUP(cudaMemset(p->part_done, 0, DFFT_MAX_PARTS * sizeof(unsigned long long)));
                }
            }
        }
    }
    {
        // stream-pipelined forward (z-parts): send side and receive side on two streams, see fwd_pipelined
        const char* env = getenv("DFFT_PIPELINE");
        // Policy (multi-GPU sweeps; not yet repeated on H100):
        //  * 2 devices: the transform is HBM / L2-fabric bound and close to its (6+2) E M roofline without overlap, and cutting
        //    it into parts was slower: never pipelined by default.
        //  * two streams (any exchange): a Y-part kernel and an X-part kernel each want both CTA slots of an SM, so they
        //    serialise or halve each other; NCCL's kernels compete for the same slots: opt-in only.
        //  * kernel chain (cubes, P2P): [Z + Y0] [Y1 + X0] ... [X last] with the two roles pinned to the two CTA slots of every SM.
        //    It paid off at 4 devices for 1024^3 and tied or lost for smaller cubes.
        //    Default from 4 devices on for axes >= 1024 points, where the X pass that it hides is long enough to pay for the
        //    extra launches and the second read of the intermediate.
        // DFFT_FORCE_PIPELINE / DFFT_PIPELINE=1 pipeline wherever it is possible, DFFT_NO_PIPELINE / DFFT_PIPELINE=0 never.
        const bool possible = P > 1 && !p->overlap && !real && !conv && (xmode == DFFT_EXCHANGE_P2P || xmode == DFFT_EXCHANGE_NCCL);
        const bool chain_ok = direction == DFFT_FORWARD && xmode == DFFT_EXCHANGE_P2P && p->fuse && ey == ex && ey->fused_yx != nullptr;
        bool want = possible && chain_ok && P >= 4 && n2 >= 1024;
        if (env) want = possible && strcmp(env, "0") != 0;
        if (flags & DFFT_FORCE_PIPELINE) want = possible;
        if (direction == DFFT_BACKWARD && getenv("DFFT_PIPELINE_BWD") && !strcmp(getenv("DFFT_PIPELINE_BWD"), "0")) want = false;
        if (flags & DFFT_NO_PIPELINE) want = false;
        if (xmode == DFFT_EXCHANGE_NCCL && (n0 % P || n1 % P)) want = false;   // ncclAlltoAll parts need equal chunks
        if (want) {
            const int cy = direction == DFFT_FORWARD ? ey->p_C : ey->s_C, cx_ = ex->x_C;
            const int m = cy > cx_ ? cy : cx_;
            int K = 0;
            if (m % cy == 0 && m % cx_ == 0) {
                for (int k : {4, 2})
                    if (n2 % ((long long)k * m) == 0 && n2 / k >= 32) { K = k; break; }
                if (getenv("DFFT_PARTS")) {
                    const int k = atoi(getenv("DFFT_PARTS"));
                    if (k >= 1 && k <= DFFT_MAX_PARTS && n2 % ((long long)k * m) == 0) K = k;
                }
            }
            if (K >= 1 && (K > 1 || getenv("DFFT_PARTS"))) {
                p->parts = K;
                p->pipe = true;
                {
                    const char* pm = getenv("DFFT_PIPE_MODE");   // "streams": the two-stream schedule even where the kernel chain is possible
                    p->pipe_fyx = direction == DFFT_FORWARD && xmode == DFFT_EXCHANGE_P2P && p->fuse && ey == ex && ey->fused_yx != nullptr &&
                                  !(pm && !strcmp(pm, "streams"));
                }
                if (dry) { p->mid = fake_addr(dev_idx, 4); p->sendbuf = fake_addr(dev_idx, 6); }
                else {
                    if (!p->mid && direction == DFFT_FORWARD) CUP(cudaMalloc(&p->mid, (size_t)p->max_count * p->esz));
                    if (xmode == DFFT_EXCHANGE_NCCL) {
                        CUP(cudaMalloc(&p->sendbuf, (size_t)p->max_count * p->esz));
                        CUP(cudaStreamCreateWithFlags(&p->stream3, cudaStreamNonBlocking));
                    }
                    if (xmode == DFFT_EXCHANGE_P2P && !getenv("DFFT_SIGNAL_KERNELS")) {
                        CUP(cudaMalloc((void**)&p->done_ctr, DFFT_MAX_PARTS * sizeof(unsigned int)));
                        CUP(cudaMemset(p->done_ctr, 0, DFFT_MAX_PARTS * sizeof(unsigned int)));
                    }
                    CUP(cudaStreamCreateWithFlags(&p->stream2, cudaStreamNonBlocking));
                    CUP(cudaEventCreateWithFlags(&p->ev_join, cudaEventDisableTiming));
                    for (auto& e : p->evb) CUP(cudaEventCreate(&e));
                    for (int k = 0; k < K; k++) {
                        CUP(cudaEventCreateWithFlags(&p->ev_y[k], cudaEventDisableTiming));
                        CUP(cudaEventCreateWithFlags(&p->ev_a[k], cudaEventDisableTiming));
                    }
                }
            }
        }
    }
    if ((real || conv) && P > 1) {
        // R2C and convolve scratch where the C2C schedules borrow `out`: the forward Z output / NCCL send buffer, the backward Y output
        if (dry) p->mid = fake_addr(dev_idx, 4);
        else CUP(cudaMalloc(&p->mid, (size_t)p->max_count * p->esz));
    }
    if (conv && P > 1 && xmode == DFFT_EXCHANGE_P2P) {
        if (dry) p->work2 = fake_addr(dev_idx, 7);
        else CUP(cudaMalloc(&p->work2, (size_t)p->max_count * p->esz));
    }
    if (P > 1 && dry) {
        p->peer_work.resize(P);
        for (int q = 0; q < P; q++) p->peer_work[q] = fake_addr(q, 3);
        if (p->work2) {
            p->peer_work2.resize(P);
            for (int q = 0; q < P; q++) p->peer_work2[q] = fake_addr(q, 7);
        }
    } else if (P > 1) {
        if (xmode == DFFT_EXCHANGE_P2P || xmode == DFFT_EXCHANGE_STAGED) {
            if (xmode == DFFT_EXCHANGE_P2P) {
                if ((rc = share_pointer(p, p->work, p->peer_work)) != 0) return bail(rc);
                if (p->work2 && (rc = share_pointer(p, p->work2, p->peer_work2)) != 0) return bail(rc);
            } else {
                if ((rc = share_pointer(p, p->buf1, p->peer_buf1)) != 0) return bail(rc);
            }
            CUP(cudaMalloc((void**)&p->sync, sizeof(SyncBlock)));
            CUP(cudaMemset(p->sync, 0, sizeof(SyncBlock)));
            if (xmode == DFFT_EXCHANGE_P2P && !p->done_ctr && !getenv("DFFT_SIGNAL_KERNELS")) {
                CUP(cudaMalloc((void**)&p->done_ctr, DFFT_MAX_PARTS * sizeof(unsigned int)));
                CUP(cudaMemset(p->done_ctr, 0, DFFT_MAX_PARTS * sizeof(unsigned int)));
            }
            std::vector<void*> ps;
            if ((rc = share_pointer(p, p->sync, ps)) != 0) return bail(rc);
            p->peer_sync.resize(P);
            for (int q = 0; q < P; q++) p->peer_sync[q] = (SyncBlock*)ps[q];
        } else {
            NcclApi& api = nccl_api();
            if (!api.ok) return bail(fail(DFFT_ECOMM, "libnccl.so.2 could not be loaded (set DFFT_NCCL_LIB)"));
            NcclUid uid;
            memset(&uid, 0, sizeof(uid));
            if (p->me == 0) {
                int r = api.GetUniqueId(&uid);
                if (r != 0) return bail(fail(DFFT_ECOMM, "ncclGetUniqueId failed"));
            }
            std::vector<NcclUid> all(P);
            if (comm->allgather(p->me, &uid, all.data(), sizeof(uid)) != 0) return bail(fail(DFFT_ECOMM, "bootstrap allgather failed"));
            int r = api.CommInitRank(&p->nccl, P, all[0], p->me);
            if (r != 0) return bail(fail(DFFT_ECOMM, "ncclCommInitRank failed: %s", api.GetErrorString ? api.GetErrorString(r) : "?"));
        }
        if (comm->host_barrier(p->me) != 0) return bail(fail(DFFT_ECOMM, "a peer failed during plan creation"));
    }
    p->stage = (real || conv) ? p->mid : p->buf2;
    p->ybwd = real ? (P == 1 ? p->work : p->mid) : p->buf2;
    if (!dry) CUP(cudaDeviceSynchronize());
#undef CUP
    *plan_out = p;
    return 0;
}

extern "C" int dfft_destroy(dfft_plan p)
{
    if (!p) return 0;
    if (p->dry) { delete p; return 0; }   // nothing was allocated
    cudaSetDevice(p->device);
    if (p->stream) cudaStreamSynchronize(p->stream);
    if (p->P > 1 && p->comm && (p->sync || p->nccl)) p->comm->host_barrier(p->me);   // nobody still writes into my buffers
    if (p->nccl) nccl_api().CommDestroy(p->nccl);
    for (void* q : p->ipc_opened) cudaIpcCloseMemHandle(q);
    if (p->P > 1 && p->comm && !p->comm->local && !p->ipc_opened.empty()) p->comm->host_barrier(p->me);
    if (p->buf1) cudaFree(p->buf1);
    if (p->work) cudaFree(p->work);
    if (p->work2) cudaFree(p->work2);
    if (p->sync) cudaFree(p->sync);
    if (p->stream2) cudaStreamSynchronize(p->stream2);
    if (p->stream3) cudaStreamSynchronize(p->stream3);
    if (p->mid) cudaFree(p->mid);
    if (p->sendbuf) cudaFree(p->sendbuf);
    if (p->done_ctr) cudaFree(p->done_ctr);
    if (p->dbg) cudaFree(p->dbg);
    if (p->ev_join) cudaEventDestroy(p->ev_join);
    for (auto& e : p->evb) if (e) cudaEventDestroy(e);
    for (auto& e : p->ev_y) if (e) cudaEventDestroy(e);
    for (auto& e : p->ev_a) if (e) cudaEventDestroy(e);
    if (p->stream2) cudaStreamDestroy(p->stream2);
    if (p->stream3) cudaStreamDestroy(p->stream3);
    if (p->part_done) cudaFree(p->part_done);
    if (p->plane_done) cudaFree(p->plane_done);
    if (p->ticket) cudaFree(p->ticket);
    if (p->lut_z) cudaFree(p->lut_z);
    if (p->lut_y) cudaFree(p->lut_y);
    if (p->lut_x) cudaFree(p->lut_x);
    if (p->lut_xn) cudaFree(p->lut_xn);
    if (p->lut_tz) cudaFree(p->lut_tz);
    if (p->lut_ty) cudaFree(p->lut_ty);
    if (p->lut_tx) cudaFree(p->lut_tx);
    for (auto& e : p->ev) if (e) cudaEventDestroy(e);
    for (auto& pe : p->pev) for (auto& e : pe) if (e) cudaEventDestroy(e);
    if (p->stream) cudaStreamDestroy(p->stream);
    cudaGetLastError();
    delete p;
    return 0;
}

extern "C" int dfft_cleanup(void) { return 0; }

extern "C" int dfft_memcpy(void* dst, const void* src, size_t bytes, int kind)
{
    CU(cudaMemcpy(dst, src, bytes, kind == 1 ? cudaMemcpyHostToDevice : (kind == 2 ? cudaMemcpyDeviceToHost : cudaMemcpyDefault)));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// pass launches
// ------------------------------------------------------------------------------------------------
// start gate / completion signal folded into a pass kernel (TileArgs::wait_flags, TileArgs::sig) instead of separate
// one-CTA launches: `which` 0 = ready[], 1 = arrive[], 2 + k = part_arrive[k]
struct Fold {
    int wait_which = -1; unsigned long long wait_val = 0;
    int sig_which = -1; unsigned long long sig_val = 0;
    int ctr = 0;     // which done_ctr word counts the finished CTAs of this launch
};
template <typename T> static void apply_fold(dfft_plan p, TileArgs<T>& a, const Fold* f)
{
    if (!f || p->dry || !p->sync) return;
    auto mine = [&](int w) -> const unsigned long long* { return w == 0 ? p->sync->ready : (w == 1 ? p->sync->arrive : p->sync->part_arrive[w - 2]); };
    if (f->wait_which >= 0 && f->wait_val > 0) { a.wait_flags = mine(f->wait_which); a.wait_val = f->wait_val; a.wait_n = p->P; }
    if (f->sig_which >= 0) {
        a.sig_n = p->P; a.sig_val = f->sig_val; a.done_ctr = p->done_ctr + f->ctr;
        for (int q = 0; q < p->P; q++) {
            SyncBlock* sb = p->peer_sync[q];
            a.sig[q] = f->sig_which == 0 ? &sb->ready[p->me] : (f->sig_which == 1 ? &sb->arrive[p->me] : &sb->part_arrive[f->sig_which - 2][p->me]);
        }
    }
}

// whether the pass of TMA mode `mode` over `extent` lines (Z) / columns (Y, X) runs on the TMA-pipelined kernel
static bool tma_ok(dfft_plan p, int mode, long long extent)
{
    const TmaEntry* e = mode == TMA_Z ? p->tz : (mode == TMA_Y ? p->ty : p->tx);
    return e && (e->use & (1u << mode)) && !p->dry && extent % e->C == 0;
}

template <typename T> struct Pass {
    // one launch: in a describe-only plan `rec` records what would run; otherwise `go` launches between the per-pass event
    // brackets of the axes ax0..ax1 it covers (none inside the pipelined schedules, which bracket their parts themselves)
    template <class Rec, class Go> static int issue(dfft_plan p, int ax0, int ax1, Rec&& rec, Go&& go, const char* what, int N)
    {
        if (p->dry) {
            rec();
            p->launches++;
            return 0;
        }
        if (!p->in_pipe) ev_record(p, p->pev[ax0][0]);
        const cudaError_t err = go();
        if (!p->in_pipe) {
            ev_record(p, p->pev[ax0][1]);
            for (int ax = ax0 + 1; ax <= ax1; ax++) { ev_record(p, p->pev[ax][0]); ev_record(p, p->pev[ax][1]); }
        }
        if (err != cudaSuccess) return fail(DFFT_ECUDA, "%s launch (N=%d) failed: %s", what, N, cudaGetErrorString(err));
        p->launches++;
        return 0;
    }
    static T scale_factor(dfft_plan p)
    {
        const Geom& g = p->g;
        return (T)(1.0 / ((double)g.n0 * (double)g.n1 * (p->r2c ? (double)p->n2r : (double)g.n2)));
    }
    // contiguous Z lines of every local plane, C lines per tile: per plane (the fused kernels' role) or as one run of n0l*N1 lines
    static void z_lines(dfft_plan p, TileArgs<T>& a, int C, bool per_plane)
    {
        const Geom& g = p->g;
        const long long nlines = per_plane ? g.n1 : p->n0l * g.n1;
        a.G = (int)cdiv(nlines, C); a.W = (int)std::min<long long>(nlines, 0x7fffffff); a.ntiles = per_plane ? p->n0l * a.G : a.G;
        a.ia = Affine{per_plane ? g.n1 * g.n2 : 0, (long long)C * g.n2, g.n2, 1}; a.oa = a.ia;
    }
    // Y columns (length N1, stride N2) of every local plane over the z-extent zk (N2: whole planes); returns the map of the
    // [x_l][y][z] side
    static Affine y_cols(dfft_plan p, TileArgs<T>& a, int C, long long zk)
    {
        const Geom& g = p->g;
        a.G = (int)cdiv(zk, C); a.W = (int)zk; a.ntiles = p->n0l * a.G;
        return Affine{g.n1 * g.n2, C, 1, g.n2};
    }
    // X columns over the z-extent zk: the [x][y_l][z'] side (row length zk) and the transposed [y_l][z][x] side; forward loads
    // the former and stores the latter, backward the reverse
    static void x_tiles(dfft_plan p, TileArgs<T>& a, int C, long long zk, bool fwd)
    {
        const Geom& g = p->g;
        a.G = (int)cdiv(zk, C); a.W = (int)zk; a.ntiles = p->n1l * a.G;
        const Affine slab{zk, C, 1, p->n1l * zk}, tr{g.n2 * g.n0, (long long)C * g.n0, g.n0, 1};
        a.ia = fwd ? slab : tr; a.oa = fwd ? tr : slab;
    }
    // chunk q = the rows of destination / source device q at base[q]: split along y (ediv yd, n1_l(q) rows of zk points per
    // plane) or along x (ediv xd, planes of zk points)
    static void chunk_table(dfft_plan p, ChunkTab& ct, bool by_y, long long zk, void* const* base)
    {
        const Geom& g = p->g;
        ct.ediv = (int)(by_y ? g.yd() : g.xd()); ct.nchunks = p->P;
        for (int q = 0; q < p->P; q++) { ct.cptr[q] = base[q]; ct.SAq[q] = by_y ? g.n1l(q) * zk : zk; }
    }
    // controls of a two-role t0 kernel: every plane's first role (GA tiles) completes before its second role (GB tiles) reads it
    static FusedCtl fused_ctl(dfft_plan p, int GA, int GB)
    {
        FusedCtl c{};
        c.plane_done = p->plane_done; c.ticket = p->ticket; c.planes = p->n0l;
        c.GA = GA; c.GB = GB;
        c.target = p->fuse_epoch += (unsigned long long)GA;
        c.lag = p->lag;
        return c;
    }
    // DRY_RUN phase of a pass: 1 = runs after the exchange has delivered this device's receive buffer (a convolve plan's
    // backward half records from 2)
    static int phase(dfft_plan p, int dir, bool after_exchange) { return (p->conv && dir == DFFT_BACKWARD ? 2 : 0) + (after_exchange ? 1 : 0); }

    static int launch(dfft_plan p, const SizeEntry* e, int kind, TileArgs<T>& a, int dir, int axis_override = -1, cudaStream_t st = nullptr)
    {
        if (!st) st = p->stream;
        a.inv = dir == DFFT_BACKWARD ? 1 : 0;
        a.gen = e->gen;
        const int axis = axis_override >= 0 ? axis_override : (kind == PK_Z ? 0 : (kind == PK_Y || kind == PK_Y_CO || kind == PK_Y_CI ? 1 : 2));
        const int C = kind_C(e, kind);
        auto rec = [&] {
            record_op<T>(p->ops, kPassNames[kind], phase(p, dir, dir == DFFT_FORWARD ? axis == 2 : axis != 2), e->N, C, kind == PK_Y_CI,
                         kind == PK_Y_CO || kind == PK_XB_CO, kind == PK_XF || kind == PK_XF_TW, a);
        };
        char what[32];
        snprintf(what, sizeof(what), "pass (kind %d)", kind);
        return issue(p, axis, axis, rec, [&] { return e->launch[kind](&a, p->sms, st); }, what, e->N);
    }
    // one TMA-pipelined pass (fft_tma.cuh).  Tensor sides are described as (base, d1, d2, s1, s2, axis): a 3-D tensor of
    // complex elements, row length `d0`, dim1/dim2 extents and element strides, transform axis = tensor dim `axis` (1 or 2)
    struct TmaTensor { void* base; long long d0, d1, d2, s1, s2; };
    static int launch_tma(dfft_plan p, const TmaEntry* e, int mode, TmaArgs<T>& a, const TmaTensor* tin, const TmaTensor* tout, int axis, int dir,
                          cudaStream_t st = nullptr)
    {
        if (!st) st = p->stream;
        alignas(64) unsigned char mi[128], mo[128];
        const int rows = e->rows;
        const TmaTensor* ts[2] = {tin, tout};
        unsigned char* ms[2] = {mi, mo};
        for (int k = 0; k < 2; k++) {
            if (!ts[k]) continue;
            const int b1 = mode == TMA_Y ? rows : 1, b2 = mode == TMA_Y ? 1 : rows;
            const int rc = tma_encode_3d(ms[k], ts[k]->base, p->prec, ts[k]->d0, ts[k]->d1, ts[k]->d2, ts[k]->s1, ts[k]->s2, e->C, b1, b2);
            if (rc != 0) return fail(DFFT_ECUDA, "cuTensorMapEncodeTiled failed (%d) for a %lldx%lldx%lld tensor", rc, ts[k]->d0, ts[k]->d1, ts[k]->d2);
        }
        a.inv = dir == DFFT_BACKWARD ? 1 : 0;
        char what[32];
        snprintf(what, sizeof(what), "TMA pass (mode %d)", mode);
        return issue(p, axis, axis, [] {}, [&] { return e->launch(mode, &a, tin ? mi : nullptr, tout ? mo : nullptr, p->sms, st); }, what, e->N);
    }
    // contiguous lines of length N2 (n0l*N1 lines), src -> dst (in place when equal)
    static int z_pass(dfft_plan p, const void* src, void* dst, bool scale, int dir)
    {
        const Geom& g = p->g;
        if (tma_ok(p, TMA_Z, p->n0l * g.n1)) {
            TmaArgs<T> t{};
            t.in = (const cx<T>*)src; t.out = (cx<T>*)dst; t.lut = (const cx<T>*)p->lut_tz;
            t.ntiles = p->n0l * g.n1 / p->tz->C; t.G = (int)std::min<long long>(t.ntiles, 0x7fffffff);
            t.in_SA = t.out_SA = (long long)t.G * p->tz->C * g.n2;   // a = tile / G: only needed beyond 2^31 tiles
            t.do_scale = scale ? 1 : 0; t.scale = scale_factor(p);
            return launch_tma(p, p->tz, TMA_Z, t, nullptr, nullptr, 0, dir);
        }
        TileArgs<T> a{};
        z_lines(p, a, p->ez->z_C, false);
        a.in = (const cx<T>*)src; a.out = (cx<T>*)dst; a.lut = (const cx<T>*)p->lut_z;
        a.do_scale = scale ? 1 : 0; a.scale = scale_factor(p);
        return launch(p, p->ez, PK_Z, a, dir);
    }
    // real-data Z pass of an R2C plan (fft_real.cuh): the n0l*N1 real lines of N2r points, two per complex transform, <-> as many
    // half-spectrum lines of nzh = g.n2 points.  Forward: src real -> dst complex; backward: src complex -> dst real (+ scale)
    static int z_real(dfft_plan p, const void* src, void* dst, bool scale, int dir)
    {
        const Geom& g = p->g;
        const bool fwd = dir == DFFT_FORWARD;
        const int C = p->ez->z_C;
        const long long nlines = p->n0l * g.n1, N = p->n2r, H = g.n2;
        RealZArgs<T> r{};
        TileArgs<T>& a = r.t;
        a.in = (const cx<T>*)src; a.out = (cx<T>*)dst; a.lut = (const cx<T>*)p->lut_z;
        a.G = (int)cdiv(cdiv(nlines, 2), C); a.ntiles = a.G; a.W = (int)std::min<long long>(nlines, 0x7fffffff);
        const Affine rmap{0, 2LL * C * N, 2 * N, 1}, cmap{0, 2LL * C * H, 2 * H, 1};   // tile, pair and point strides of each side
        a.ia = fwd ? rmap : cmap; a.oa = fwd ? cmap : rmap;
        r.ld_in = fwd ? N : H; r.ld_out = fwd ? H : N;   // the kernel derives nzh = N/2 + 1 from its schedule
        if (fwd) r.rin = (const T*)src;
        else r.rout = (T*)dst;
        a.inv = fwd ? 0 : 1;
        a.do_scale = scale ? 1 : 0; a.scale = scale_factor(p);
        const int kind = fwd ? PK_Z_R2C : PK_Z_C2R;
        auto rec = [&] {
            // real-side maps are in real elements; "pair" = distance between the two lines of a pair (input side, output side)
            char extra[128];
            snprintf(extra, sizeof(extra), ", \"nzh\": %lld, \"pair\": [%lld, %lld]", H, r.ld_in, r.ld_out);
            record_op<T>(p->ops, kPassNames[kind], phase(p, dir, !fwd), (int)N, C, false, false, false, a, extra);
        };
        return issue(p, 0, 0, rec, [&] { return p->ez->launch[kind](&r, p->sms, p->stream); }, "real Z pass", (int)N);
    }
    // columns of length N1 (stride N2) of every local plane.  mode 0: src -> dst natural (in place when equal)
    // mode 1: chunked (packed / peer) store, mode 2: chunked (unpack) load
    static int y_pass(dfft_plan p, const void* src, void* dst, int mode, void* const* chunk_base, const Fold* fold, int dir)
    {
        const Geom& g = p->g;
        if (mode == 0 && tma_ok(p, TMA_Y, g.n2)) {
            TmaArgs<T> t{};
            t.lut = (const cx<T>*)p->lut_ty;
            t.G = (int)(g.n2 / p->ty->C); t.ntiles = p->n0l * t.G;
            TmaTensor ti{(void*)src, g.n2, g.n1, p->n0l, g.n2, g.n1 * g.n2}, to{dst, g.n2, g.n1, p->n0l, g.n2, g.n1 * g.n2};
            return launch_tma(p, p->ty, TMA_Y, t, &ti, &to, 1, dir);
        }
        TileArgs<T> a{};
        a.in = (const cx<T>*)src; a.out = (cx<T>*)dst; a.lut = (const cx<T>*)p->lut_y;
        const int kind = mode == 0 ? PK_Y : (mode == 1 ? PK_Y_CO : PK_Y_CI);
        a.ia = a.oa = y_cols(p, a, kind_C(p->ey, kind), g.n2);
        if (mode != 0) chunk_table(p, mode == 1 ? a.co : a.ci, true, g.n2, chunk_base);
        apply_fold<T>(p, a, fold);
        return launch(p, p->ey, kind, a, dir);
    }
    // t0 in one persistent kernel (square planes): forward Z (zsrc -> mid) then Y (mid -> ydst, or chunked);
    // backward Y (ysrc or chunked -> mid) then Z (mid -> mid).  ymode as in y_pass.
    static int zy_fused(dfft_plan p, const void* src, void* mid, void* dst, int ymode, void* const* chunk_base, bool scale, const Fold* fold, int dir)
    {
        const Geom& g = p->g;
        const SizeEntry* e = p->ez;
        const bool fwd = dir == DFFT_FORWARD;
        TileArgs<T> z{}, y{};
        const int CZ = (fwd && ymode == 1) ? e->f_zCp : e->f_zC, CY = (fwd && ymode == 1) ? e->p_C : e->s_C;
        z.lut = (const cx<T>*)p->lut_z; y.lut = (const cx<T>*)p->lut_y;
        z.inv = y.inv = fwd ? 0 : 1;
        z_lines(p, z, CZ, true);   // contiguous role, tiled per plane: tile (plane, b) = CZ lines starting at line b*CZ of the plane
        z.do_scale = scale ? 1 : 0; z.scale = scale_factor(p);
        y.ia = y.oa = y_cols(p, y, CY, g.n2);
        if (ymode != 0) chunk_table(p, ymode == 1 ? y.co : y.ci, true, g.n2, chunk_base);
        if (fwd) { z.in = (const cx<T>*)src; z.out = (cx<T>*)mid; y.in = (const cx<T>*)mid; y.out = (cx<T>*)dst; }
        else { y.in = (const cx<T>*)src; y.out = (cx<T>*)mid; z.in = (const cx<T>*)mid; z.out = (cx<T>*)mid; }
        FusedCtl c = fused_ctl(p, fwd ? z.G : y.G, fwd ? y.G : z.G);
        const int kind = fwd ? (ymode == 1 ? FK_ZY_CO : FK_ZY) : (ymode == 2 ? FK_YZ_CI : FK_YZ);
        apply_fold<T>(p, fwd ? y : z, fold);   // fft_fused2_kernel gates on / signals through its second role's arguments
        auto rec = [&] {
            const int ph = phase(p, dir, !fwd);
            if (fwd) { record_op<T>(p->ops, "fusedZ", ph, e->N, CZ, false, false, false, z); record_op<T>(p->ops, "fusedY", ph, e->N, CY, false, ymode == 1, false, y); }
            else { record_op<T>(p->ops, "fusedY", ph, e->N, CY, ymode == 2, false, false, y); record_op<T>(p->ops, "fusedZ", ph, e->N, CZ, false, false, false, z); }
        };
        auto go = [&] { return fwd ? e->fused[kind](&z, &y, &c, p->sms, p->stream) : e->fused[kind](&y, &z, &c, p->sms, p->stream); };
        return issue(p, 0, 1, rec, go, "fused t0", e->N);
    }
    // forward t0 of one device in one TMA-pipelined kernel (square planes): Z: src -> mid, Y: mid -> mid in place
    static int zy_fused_tma(dfft_plan p, const void* src, void* mid)
    {
        const Geom& g = p->g;
        const TmaEntry* e = p->tz;
        alignas(64) unsigned char mm[128];
        const int rc = tma_encode_3d(mm, mid, p->prec, g.n2, g.n1, p->n0l, g.n2, g.n1 * g.n2, e->C, e->rows, 1);   // y_pass's map
        if (rc != 0) return fail(DFFT_ECUDA, "cuTensorMapEncodeTiled failed (%d) for a %lldx%lldx%lld tensor", rc, g.n2, g.n1, p->n0l);
        TmaFusedArgs<T> a{};
        a.src = (const cx<T>*)src; a.mid = (cx<T>*)mid; a.lut = (const cx<T>*)p->lut_tz;
        FusedCtl c = fused_ctl(p, (int)(g.n1 / e->C), (int)(g.n2 / e->C));
        return issue(p, 0, 1, [] {}, [&] { return e->fused_zy(&a, &c, mm, p->sms, p->stream); }, "TMA fused t0", e->N);
    }
    // forward t0 + t1 + t2 + t3 in one kernel (P2P, square planes): Z: buf1 -> mid, Y: mid -> peers' work, X: work -> buf2
    static int fwd_overlapped(dfft_plan p, void* const* peer_base)
    {
        const Geom& g = p->g;
        const SizeEntry* e = p->ez;
        TileArgs<T> z{}, y{}, x{};
        const int CZ = e->f_zCp, CY = e->p_C, CX = e->x_C;
        z.lut = (const cx<T>*)p->lut_z; y.lut = (const cx<T>*)p->lut_y; x.lut = (const cx<T>*)p->lut_x;
        z_lines(p, z, CZ, true);
        z.in = (const cx<T>*)p->buf1; z.out = (cx<T>*)p->mid;
        y.ia = y.oa = y_cols(p, y, CY, g.n2);
        y.in = (const cx<T>*)p->mid; y.out = nullptr;
        chunk_table(p, y.co, true, g.n2, peer_base);
        x_tiles(p, x, CX, g.n2, true);
        x.in = (const cx<T>*)p->work; x.out = (cx<T>*)p->buf2;
        Fused3Ctl c{};
        c.plane_done = p->plane_done; c.ticket = p->ticket; c.part_done = p->part_done;
        c.planes = p->n0l; c.rows = p->n1l; c.P = p->P; c.me = p->me;
        c.K = p->parts;
        c.GA = z.G; c.GB = y.G; c.GBk = y.G / c.K; c.GX = x.G; c.GXk = x.G / c.K;
        c.target = p->fuse_epoch += (unsigned long long)c.GA;
        c.epoch = ++p->overlap_epoch;
        c.part_target = c.epoch * (unsigned long long)(p->n0l * c.GBk);
        if (!p->dry) {
            c.my_arrive = &p->sync->part_arrive[0][0];
            for (int q = 0; q < p->P; q++) c.peer_arrive[q] = &p->peer_sync[q]->part_arrive[0][0];
        }
        c.lag = p->lag;
        c.dbg = nullptr;
        if (!p->dry && getenv("DFFT_DEBUG_TIMELINE")) {
            if (!p->dbg) cudaMalloc((void**)&p->dbg, 16 * sizeof(unsigned long long));
            cudaMemsetAsync(p->dbg, 0xff, 4 * sizeof(unsigned long long), p->stream);
            cudaMemsetAsync(p->dbg + 4, 0, 12 * sizeof(unsigned long long), p->stream);
            c.dbg = p->dbg;
        }
        auto rec = [&] {
            record_op<T>(p->ops, "ovlZ", 0, e->N, CZ, false, false, false, z);
            record_op<T>(p->ops, "ovlY", 0, e->N, CY, false, true, false, y);
            record_op<T>(p->ops, "ovlX", 1, e->N, CX, false, false, true, x);
        };
        return issue(p, 0, 2, rec, [&] { return e->fused3(&z, &y, &x, &c, p->sms, p->stream); }, "overlapped forward", e->N);
    }
    // X transform that keeps the natural [x][y][z] layout (single device): columns along x, stride N1*N2, src -> dst
    static int x_natural(dfft_plan p, const void* src, void* dst)
    {
        const Geom& g = p->g;
        TileArgs<T> a{};
        const int C = p->ex->s_C;
        a.in = (const cx<T>*)src; a.out = (cx<T>*)dst; a.lut = (const cx<T>*)p->lut_xn;
        a.G = (int)cdiv(g.n2, C); a.W = (int)g.n2; a.ntiles = g.n1 * a.G;
        a.ia = Affine{g.n2, C, 1, g.n1 * g.n2}; a.oa = a.ia;
        return launch(p, p->ex, PK_Y, a, p->direction, 2);   // a strided-local kernel, timed as the X pass
    }
    // forward X: src = [x][y_l][z] -> dst = [y_l][z][x]
    static bool x_fwd_folds(dfft_plan p) { return !tma_ok(p, TMA_XF, p->g.n2); }
    static int x_fwd(dfft_plan p, const void* src, void* dst, const Fold* fold = nullptr)
    {
        const Geom& g = p->g;
        if (tma_ok(p, TMA_XF, g.n2)) {
            TmaArgs<T> t{};
            t.lut = (const cx<T>*)p->lut_tx; t.out = (cx<T>*)dst;
            t.G = (int)(g.n2 / p->tx->C); t.ntiles = p->n1l * t.G; t.out_SA = g.n2 * g.n0;
            TmaTensor ti{(void*)src, g.n2, p->n1l, g.n0, g.n2, p->n1l * g.n2};
            return launch_tma(p, p->tx, TMA_XF, t, &ti, nullptr, 2, DFFT_FORWARD);
        }
        TileArgs<T> a{};
        x_tiles(p, a, p->ex->x_C, g.n2, true);
        a.in = (const cx<T>*)src; a.out = (cx<T>*)dst; a.lut = (const cx<T>*)p->lut_x;
        apply_fold<T>(p, a, fold);
        return launch(p, p->ex, PK_XF, a, DFFT_FORWARD);
    }
    // ---- z-part variants (stream-pipelined forward): part k of K covers the columns z in [k*zk, (k+1)*zk) ----------
    // Y pass of one z-part: mid[x_l][y][z in part] -> chunk q (the rows of destination device q) at chunk_base[q], laid out
    // [x_l][y_l(q)][z'] with row length zk: the part-major receive (P2P) / send (NCCL) layout
    static void y_part_args(dfft_plan p, TileArgs<T>& a, const void* src, long long zk, int k, void* const* chunk_base, int C)
    {
        a.in = (const cx<T>*)src + k * zk; a.out = nullptr; a.lut = (const cx<T>*)p->lut_y;
        a.ia = y_cols(p, a, C, zk);
        a.oa = Affine{0, C, 1, zk};
        chunk_table(p, a.co, true, zk, chunk_base);
        if (p->xmode == DFFT_EXCHANGE_P2P && !p->dry && p->done_ctr) {
            // the kernel's last CTA publishes "part k of sender me has arrived" (epoch) on every receiving device
            a.sig_n = p->P; a.sig_val = p->epoch; a.done_ctr = p->done_ctr + k;
            for (int q = 0; q < p->P; q++) a.sig[q] = &p->peer_sync[q]->part_arrive[k][p->me];
        }
    }
    static int y_part(dfft_plan p, const void* src, long long zk, int k, void* const* chunk_base, int cap)
    {
        TileArgs<T> a{};
        y_part_args(p, a, src, zk, k, chunk_base, p->ey->p_C);
        a.max_ctas_per_sm = cap;
        return launch(p, p->ey, PK_Y_CO, a, DFFT_FORWARD);
    }
    // part 0 together with the Z pass of every plane in one persistent kernel (fft_fused2_kernel): Z: src -> mid (L2),
    // Y part 0: mid -> chunks
    static int zy_fused_part0(dfft_plan p, const void* src, void* mid, long long zk, void* const* chunk_base)
    {
        const SizeEntry* e = p->ez;
        TileArgs<T> z{}, y{};
        const int CZ = e->f_zCp, CY = e->p_C;
        z.lut = (const cx<T>*)p->lut_z;
        z_lines(p, z, CZ, true);
        z.in = (const cx<T>*)src; z.out = (cx<T>*)mid;
        y_part_args(p, y, mid, zk, 0, chunk_base, CY);
        FusedCtl c = fused_ctl(p, z.G, y.G);
        auto rec = [&] {
            record_op<T>(p->ops, "fusedZ", 0, e->N, CZ, false, false, false, z);
            record_op<T>(p->ops, "fusedY", 0, e->N, CY, false, true, false, y);
        };
        return issue(p, 0, 1, rec, [&] { return e->fused[FK_ZY_CO](&z, &y, &c, p->sms, p->stream); }, "fused t0 (part 0)", e->N);
    }
    // X pass of one z-part on the receive side: rpart = [x (all N0)][y_l][z'] (row length zk) -> dst[y_l][z in part][x]
    static void x_part_args(dfft_plan p, TileArgs<T>& a, const void* rpart, void* dst, long long zk, int k)
    {
        x_tiles(p, a, p->ex->x_C, zk, true);
        a.in = (const cx<T>*)rpart; a.out = (cx<T>*)dst + k * zk * p->g.n0; a.lut = (const cx<T>*)p->lut_x;
    }
    // Y pass of part k (stores to the peers) and X pass of part k-1 (already arrived) in one two-role kernel
    static int yx_fused(dfft_plan p, const void* mid, long long zk, int k, void* const* chunk_base, const void* rpart_prev, void* dst)
    {
        const SizeEntry* e = p->ey;
        TileArgs<T> y{}, x{};
        y_part_args(p, y, mid, zk, k, chunk_base, e->p_C);
        x_part_args(p, x, rpart_prev, dst, zk, k - 1);
        YxCtl c{};
        c.ticket = p->ticket;
        c.TA = (unsigned)y.ntiles; c.TB = (unsigned)x.ntiles;
        auto rec = [&] {
            record_op<T>(p->ops, "Y_CO", 0, e->N, e->p_C, false, true, false, y);
            record_op<T>(p->ops, "XF", 1, e->N, e->x_C, false, false, true, x);
        };
        return issue(p, 1, 2, rec, [&] { return e->fused_yx(&y, &x, &c, p->sms, p->stream); }, "fused Y+X part", e->N);
    }
    static int x_part(dfft_plan p, const void* rpart, void* dst, long long zk, int k, int cap, cudaStream_t st)
    {
        const Geom& g = p->g;
        // the TMA kernel takes the whole SM (one CTA, 3-slot ring): only for a part that overlaps nothing (the last one)
        if (cap == 0 && tma_ok(p, TMA_XF, zk)) {
            TmaArgs<T> t{};
            t.lut = (const cx<T>*)p->lut_tx; t.out = (cx<T>*)dst + k * zk * g.n0;
            t.G = (int)(zk / p->tx->C); t.ntiles = p->n1l * t.G; t.out_SA = g.n2 * g.n0;
            TmaTensor ti{(void*)rpart, zk, p->n1l, g.n0, zk, p->n1l * zk};
            return launch_tma(p, p->tx, TMA_XF, t, &ti, nullptr, 2, DFFT_FORWARD, st);
        }
        TileArgs<T> a{};
        x_part_args(p, a, rpart, dst, zk, k);
        a.max_ctas_per_sm = cap;
        return launch(p, p->ex, PK_XF, a, DFFT_FORWARD, -1, st);
    }
    // ---- z-part variants of the BACKWARD passes (stream-pipelined backward) --------------------------------------------------
    // inverse X pass of one z-part: src[y_l][z in part][x] -> chunk p (= the x-planes of destination device p) at chunk_base[p],
    // laid out [x_l][y_l][z'] with row length zk
    static int xb_part(dfft_plan p, const void* src, long long zk, int k, void* const* chunk_base, int cap)
    {
        TileArgs<T> a{};
        x_tiles(p, a, p->ex->xo_C, zk, false);
        a.oa.SA = 0;   // the chunk table's SAq places the planes
        a.in = (const cx<T>*)src + k * zk * p->g.n0; a.out = nullptr; a.lut = (const cx<T>*)p->lut_x;
        chunk_table(p, a.co, false, zk, chunk_base);
        if (p->xmode == DFFT_EXCHANGE_P2P && !p->dry && p->done_ctr) {
            a.sig_n = p->P; a.sig_val = p->epoch; a.done_ctr = p->done_ctr + k;
            for (int q = 0; q < p->P; q++) a.sig[q] = &p->peer_sync[q]->part_arrive[k][p->me];
        }
        a.max_ctas_per_sm = cap;
        return launch(p, p->ex, PK_XB_CO, a, DFFT_BACKWARD);
    }
    // inverse Y pass of one z-part on the receive side: rpart = [sender q][x_l][y_l(q)][z'] -> dst[x_l][y][z in part]
    static void yinv_part_args(dfft_plan p, TileArgs<T>& a, const void* rpart, void* dst, long long zk, int k, int C)
    {
        const Geom& g = p->g;
        a.in = nullptr; a.out = (cx<T>*)dst + k * zk; a.lut = (const cx<T>*)p->lut_y;
        a.oa = y_cols(p, a, C, zk);
        a.ia = Affine{0, C, 1, zk};
        void* base[DFFT_MAX_CHUNKS];
        for (int q = 0; q < p->P; q++) base[q] = eoff((void*)rpart, (long long)q * p->n0l * g.yd() * zk, p->esz);
        chunk_table(p, a.ci, true, zk, base);
    }
    static int yinv_part(dfft_plan p, const void* rpart, void* dst, long long zk, int k, int cap, cudaStream_t st)
    {
        TileArgs<T> a{};
        yinv_part_args(p, a, rpart, dst, zk, k, p->ey->ci_C);
        a.max_ctas_per_sm = cap;
        return launch(p, p->ey, PK_Y_CI, a, DFFT_BACKWARD, -1, st);
    }
    // the LAST part's inverse Y pass completes every plane: it runs fused with the inverse Z pass (fft_fused2_kernel, Y then Z)
    static int yz_fused_last_part(dfft_plan p, const void* rpart, void* dst, long long zk, int k, bool scale, cudaStream_t st)
    {
        const SizeEntry* e = p->ez;
        TileArgs<T> z{}, y{};
        const int CZ = e->f_zC, CY = e->s_C;
        yinv_part_args(p, y, rpart, dst, zk, k, CY);
        y.inv = 1;
        z.lut = (const cx<T>*)p->lut_z; z.inv = 1;
        z_lines(p, z, CZ, true);
        z.in = (const cx<T>*)dst; z.out = (cx<T>*)dst;
        z.do_scale = scale ? 1 : 0; z.scale = scale_factor(p);
        FusedCtl c = fused_ctl(p, y.G, z.G);
        auto rec = [&] {
            record_op<T>(p->ops, "fusedY", 1, e->N, CY, true, false, false, y);
            record_op<T>(p->ops, "fusedZ", 1, e->N, CZ, false, false, false, z);
        };
        return issue(p, 0, 1, rec, [&] { return e->fused[FK_YZ_CI](&y, &z, &c, p->sms, st); }, "fused inverse t0 (last part)", e->N);
    }
    // backward X: src = [y_l][z][x] -> dst = [x][y_l][z] (chunked by destination device when chunk_base)
    static int x_bwd(dfft_plan p, const void* src, void* dst, void* const* chunk_base, const Fold* fold = nullptr)
    {
        const Geom& g = p->g;
        if (!chunk_base && tma_ok(p, TMA_XB, g.n2)) {
            TmaArgs<T> t{};
            t.lut = (const cx<T>*)p->lut_tx; t.in = (const cx<T>*)src;
            t.G = (int)(g.n2 / p->tx->C); t.ntiles = p->n1l * t.G; t.in_SA = g.n2 * g.n0;
            TmaTensor to{dst, g.n2, p->n1l, g.n0, g.n2, p->n1l * g.n2};
            return launch_tma(p, p->tx, TMA_XB, t, nullptr, &to, 2, DFFT_BACKWARD);
        }
        TileArgs<T> a{};
        x_tiles(p, a, chunk_base ? p->ex->xo_C : p->ex->x_C, g.n2, false);
        a.in = (const cx<T>*)src; a.out = (cx<T>*)dst; a.lut = (const cx<T>*)p->lut_x;
        if (chunk_base) {
            chunk_table(p, a.co, false, g.n2, chunk_base);
            apply_fold<T>(p, a, fold);
        }
        return launch(p, p->ex, chunk_base ? PK_XB_CO : PK_XB, a, DFFT_BACKWARD);
    }
    // fused X pass of a convolve plan (fft_conv_kernel): the [x][y_l][z'] columns of src, transformed along x, multiplied by
    // mult (same layout), transformed back -> dst in the same layout, or (chunk_base) split by xd into the destinations' receive
    // buffers [x_l][y_l(me)][z'] as x_bwd's chunked store does.  DFFT_SCALE_BACKWARD's 1/N rides on the multiply
    static int x_conv(dfft_plan p, const void* src, void* dst, void* const* chunk_base, const void* mult, const Fold* fold)
    {
        const Geom& g = p->g;
        const bool co = chunk_base != nullptr;
        const int kind = co ? PK_XCONV_CO : PK_XCONV;
        const int C = kind_C(p->ex, kind);
        ConvArgs<T> r{};
        TileArgs<T>& a = r.t;
        a.in = (const cx<T>*)src; a.out = (cx<T>*)dst; a.lut = (const cx<T>*)p->lut_xn;
        x_tiles(p, a, C, g.n2, true);
        a.oa = a.ia;
        a.do_scale = (p->flags & DFFT_SCALE_BACKWARD) ? 1 : 0; a.scale = scale_factor(p);
        if (co) chunk_table(p, a.co, false, g.n2, chunk_base);
        r.mult = (const cx<T>*)mult;
        apply_fold<T>(p, a, fold);
        auto rec = [&] {
            char extra[64];
            snprintf(extra, sizeof(extra), ", \"mult\": %llu", (unsigned long long)(size_t)mult);
            record_op<T>(p->ops, kPassNames[kind], 1, p->ex->N, C, false, co, false, a, extra);
        };
        return issue(p, 2, 2, rec, [&] { return p->ex->launch[kind](&r, p->sms, p->stream); }, "convolution X pass", p->ex->N);
    }
};

// exchange offsets (api.cpp:84-133, 613-627): where chunk (sender s -> receiver r) starts
static long long send_off(const Geom& g, int s, int r, int dir)
{
    return dir == DFFT_FORWARD ? (long long)r * g.n0l(s) * g.yd() * g.n2 : (long long)r * g.xd() * g.n1l(s) * g.n2;
}
static long long recv_off(const Geom& g, int s, int r, int dir)
{
    return dir == DFFT_FORWARD ? (long long)s * g.xd() * g.n1l(r) * g.n2 : (long long)s * g.n0l(r) * g.yd() * g.n2;
}
static long long xchg_count(const Geom& g, int s, int r, int dir)
{
    return dir == DFFT_FORWARD ? g.n0l(s) * g.n1l(r) * g.n2 : g.n0l(r) * g.n1l(s) * g.n2;
}

/* the reference's TransInfo table (fft_mpi_common.h:24-29, filled at api.cpp:84-133) */
extern "C" int dfft_exchange_table(long long n0, long long n1, long long n2, int P, int dev, int direction, long long* scount,
                                   long long* soffset, long long* rcount, long long* roffset)
{
    if (P < 1 || dev < 0 || dev >= P || (direction != DFFT_FORWARD && direction != DFFT_BACKWARD)) return fail(DFFT_EINVAL, "bad arguments");
    Geom g{n0, n1, n2, P};
    if (g.last_n0() < 1 || g.last_n1() < 1) return fail(DFFT_EUNSUPPORTED, "empty last slab");
    for (int i = 0; i < P; i++) {
        if (scount) scount[i] = xchg_count(g, dev, i, direction);
        if (soffset) soffset[i] = send_off(g, dev, i, direction);
        if (rcount) rcount[i] = xchg_count(g, i, dev, direction);
        if (roffset) roffset[i] = recv_off(g, i, dev, direction);
    }
    return 0;
}

// which: 0 = ready[], 1 = arrive[], 2 + k = part_arrive[k][]
static int flags_signal(dfft_plan p, int which, unsigned long long value, cudaStream_t st = nullptr)
{
    if (p->dry) return 0;
    FlagPtrs fp{};
    for (int q = 0; q < p->P; q++) {
        SyncBlock* sb = p->peer_sync[q];
        fp.p[q] = which == 1 ? &sb->arrive[p->me] : (which == 0 ? &sb->ready[p->me] : &sb->part_arrive[which - 2][p->me]);
    }
    signal_flags_kernel<<<1, DFFT_MAX_CHUNKS, 0, st ? st : p->stream>>>(fp, p->P, value);
    CU(cudaGetLastError());
    p->launches++;
    return 0;
}
static int flags_wait(dfft_plan p, int which, unsigned long long value, cudaStream_t st = nullptr)
{
    if (value == 0 || p->dry) return 0;
    const unsigned long long* f = which == 1 ? p->sync->arrive : (which == 0 ? p->sync->ready : p->sync->part_arrive[which - 2]);
    wait_flags_kernel<<<1, DFFT_MAX_CHUNKS, 0, st ? st : p->stream>>>(f, p->P, value);
    CU(cudaGetLastError());
    p->launches++;
    return 0;
}

static int nccl_exchange(dfft_plan p, const void* sendbuf, void* recvbuf, int dir)
{
    const Geom& g = p->g;
    if (p->dry) {   // describe the all-to-all: element offsets and counts of every chunk this device sends
        char buf[160];
        std::string o = "{\"op\": \"alltoall\", \"phase\": " + std::to_string(p->conv && dir == DFFT_BACKWARD ? 2 : 0) + ", ";
        snprintf(buf, sizeof(buf), "\"send\": %llu, \"recv\": %llu, \"esz\": %zu, \"chunks\": [", (unsigned long long)(size_t)sendbuf,
                 (unsigned long long)(size_t)recvbuf, p->esz);
        o += buf;
        for (int q = 0; q < p->P; q++) {
            snprintf(buf, sizeof(buf), "%s[%d, %lld, %lld, %lld]", q ? ", " : "", q, send_off(g, p->me, q, dir), recv_off(g, p->me, q, dir), xchg_count(g, p->me, q, dir));
            o += buf;
        }
        o += "]}";
        p->ops.push_back(o);
        p->launches++;
        return 0;
    }
    NcclApi& api = nccl_api();
    bool even = true;
    for (int q = 0; q < p->P; q++)
        if (xchg_count(g, p->me, q, dir) != xchg_count(g, 0, 0, dir) || xchg_count(g, q, p->me, dir) != xchg_count(g, 0, 0, dir)) even = false;
    if (even && api.AlltoAll && !getenv("DFFT_NCCL_SENDRECV")) {
        NC(api.AlltoAll(sendbuf, recvbuf, (size_t)xchg_count(g, 0, 0, dir) * p->esz, /*ncclInt8*/ 0, p->nccl, p->stream));
    } else {
        NC(api.GroupStart());
        for (int q = 0; q < p->P; q++) {
            NC(api.Send(eoff((void*)sendbuf, send_off(g, p->me, q, dir), p->esz), (size_t)xchg_count(g, p->me, q, dir) * p->esz, 0, q, p->nccl, p->stream));
            NC(api.Recv(eoff(recvbuf, recv_off(g, q, p->me, dir), p->esz), (size_t)xchg_count(g, q, p->me, dir) * p->esz, 0, q, p->nccl, p->stream));
        }
        NC(api.GroupEnd());
    }
    p->launches++;
    return 0;
}

// one z-part of the all-to-all in NCCL mode (even split): `count` elements to / from every device, chunk q of the send
// part at q*count, the chunk received from device s at s*count of the receive part
static int nccl_exchange_part(dfft_plan p, const void* sendpart, void* recvpart, long long count, cudaStream_t st)
{
    if (p->dry) {
        char buf[160];
        std::string o = "{\"op\": \"alltoall\", \"phase\": 0, ";
        snprintf(buf, sizeof(buf), "\"send\": %llu, \"recv\": %llu, \"esz\": %zu, \"chunks\": [", (unsigned long long)(size_t)sendpart,
                 (unsigned long long)(size_t)recvpart, p->esz);
        o += buf;
        for (int q = 0; q < p->P; q++) {
            snprintf(buf, sizeof(buf), "%s[%d, %lld, %lld, %lld]", q ? ", " : "", q, (long long)q * count, (long long)p->me * count, count);
            o += buf;
        }
        o += "]}";
        p->ops.push_back(o);
        p->launches++;
        return 0;
    }
    NcclApi& api = nccl_api();
    if (api.AlltoAll && !getenv("DFFT_NCCL_SENDRECV")) {
        NC(api.AlltoAll(sendpart, recvpart, (size_t)count * p->esz, /*ncclInt8*/ 0, p->nccl, st));
    } else {
        NC(api.GroupStart());
        for (int q = 0; q < p->P; q++) {
            NC(api.Send(eoff((void*)sendpart, (long long)q * count, p->esz), (size_t)count * p->esz, 0, q, p->nccl, st));
            NC(api.Recv(eoff(recvpart, (long long)q * count, p->esz), (size_t)count * p->esz, 0, q, p->nccl, st));
        }
        NC(api.GroupEnd());
    }
    p->launches++;
    return 0;
}

// Stream-pipelined forward transform (P > 1).  The reference runs t0, t1, t2, t3 back to back with a device-wide sync
// after each (fft_mpi_3d_api.cpp:181-201, 610-672: no overlap at all).  Here the z axis is cut into K parts:
//   send side, plan stream    : Z pass of the slab (fused with Y part 0 through L2 when the planes are square), then for
//                               every part k the Y pass of its columns, whose store IS the pack (t1) and -- P2P -- the
//                               all-to-all (t2): rows go straight into the peers' receive buffers over NVLink, followed by a
//                               per-part arrival flag.  NCCL: the packed part is handed to ncclAlltoAll on the comm stream.
//   receive side, second stream: as soon as part k has arrived from every sender, the X pass of the (y_l, z in part k)
//                               lines (t3, unpack + transpose folded into its load / store), while later parts are still
//                               being computed and sent.
// Both sides cap their resident CTAs per SM while they overlap so that they co-reside on every SM.
// Receive / send buffers are part-major: part k of device q = [x (all N0)][y_l][z'] with z' < zk at k * N0 * n1_l(q) * zk.
template <typename T> static int fwd_pipelined(dfft_plan p)
{
    const Geom& g = p->g;
    const int P = p->P, me = p->me, K = p->parts;
    const long long zk = g.n2 / K;
    const bool p2p = p->xmode == DFFT_EXCHANGE_P2P;
    cudaStream_t A = p->stream, B = p->stream2, Cs = p->stream3;
    int rc = 0;
    struct Guard { dfft_plan p; ~Guard() { p->in_pipe = false; } } guard{p};
    p->in_pipe = true;
    int cap = 1;
    if (getenv("DFFT_PIPE_CAP")) cap = atoi(getenv("DFFT_PIPE_CAP"));
    if (p2p) {
        p->epoch++;
        if ((rc = flags_wait(p, 0, p->epoch - 1))) return rc;   // every receiver has consumed the previous epoch
    }
    CU(ev_record(p, p->pev[0][0]));
    if (p->pipe_fyx) {
        // chain of two-role kernels on the plan stream: [Z + Y part 0] [Y part 1 + X part 0] ... [Y part K-1 + X part K-2] [X part K-1]
        for (int k = 0; k < K; k++) {
            void* base[DFFT_MAX_CHUNKS];
            for (int q = 0; q < P; q++) base[q] = eoff(p->peer_work[q], ((long long)k * g.n0 + (long long)me * g.xd()) * g.n1l(q) * zk, p->esz);
            if (k == 0) rc = Pass<T>::zy_fused_part0(p, p->buf1, p->mid, zk, base);
            else {
                // part k-1 must have arrived from every sender before the kernel whose X role consumes it starts: a one-CTA gate
                // kernel, not a poll inside the full-grid kernel (which would hold every SM slot while it waits, see execute_slabs)
                if ((rc = flags_wait(p, 2 + k - 1, p->epoch, A))) return rc;
                rc = Pass<T>::yx_fused(p, p->mid, zk, k, base, eoff(p->work, (long long)(k - 1) * g.n0 * p->n1l * zk, p->esz), p->buf2);
            }
            if (rc) return rc;
            if (!p->done_ctr && (rc = flags_signal(p, 2 + k, p->epoch, A))) return rc;   // else the kernel's last CTA publishes the flags
        }
        CU(ev_record(p, p->pev[0][1]));
        CU(ev_record(p, p->pev[1][0])); CU(ev_record(p, p->pev[1][1]));
        CU(ev_record(p, p->ev[1]));
        if ((rc = flags_wait(p, 2 + K - 1, p->epoch, A))) return rc;
        CU(ev_record(p, p->evb[0]));
        CU(ev_record(p, p->pev[2][0]));
        if ((rc = Pass<T>::x_part(p, eoff(p->work, (long long)(K - 1) * g.n0 * p->n1l * zk, p->esz), p->buf2, zk, K - 1, 0, A))) return rc;
        CU(ev_record(p, p->pev[2][1]));
        CU(ev_record(p, p->evb[1]));
        if ((rc = flags_signal(p, 0, p->epoch, A))) return rc;
        CU(ev_record(p, p->ev[2]));
        CU(ev_record(p, p->ev[3]));
        p->timed = true;
        return 0;
    }
    for (int k = 0; k < K; k++) {
        void* base[DFFT_MAX_CHUNKS];
        for (int q = 0; q < P; q++)
            base[q] = p2p ? eoff(p->peer_work[q], ((long long)k * g.n0 + (long long)me * g.xd()) * g.n1l(q) * zk, p->esz)
                          : eoff(p->sendbuf, ((long long)k * P + q) * p->n0l * g.yd() * zk, p->esz);
        if (k == 0 && p->fuse) rc = Pass<T>::zy_fused_part0(p, p->buf1, p->mid, zk, base);
        else {
            if (k == 0 && (rc = Pass<T>::z_pass(p, p->buf1, p->mid, false, DFFT_FORWARD))) return rc;
            rc = Pass<T>::y_part(p, p->mid, zk, k, base, k > 0 ? cap : 0);
        }
        if (rc) return rc;
        if (p2p) {
            if (!p->done_ctr && (rc = flags_signal(p, 2 + k, p->epoch, A))) return rc;   // else folded into the part kernel
        } else {
            const long long chunk = p->n0l * g.yd() * zk;
            CU(ev_record_on(p, p->ev_y[k], A));
            CU(stream_wait(p, Cs, p->ev_y[k]));
            if ((rc = nccl_exchange_part(p, eoff(p->sendbuf, (long long)k * P * chunk, p->esz), eoff(p->work, (long long)k * P * chunk, p->esz), chunk, Cs))) return rc;
            CU(ev_record_on(p, p->ev_a[k], Cs));
        }
    }
    CU(ev_record(p, p->pev[0][1]));
    CU(ev_record(p, p->pev[1][0]));
    CU(ev_record(p, p->pev[1][1]));
    CU(ev_record(p, p->ev[1]));
    for (int k = 0; k < K; k++) {
        if (p2p) { if ((rc = flags_wait(p, 2 + k, p->epoch, B))) return rc; }
        else CU(stream_wait(p, B, p->ev_a[k]));
        if (k == 0) CU(ev_record_on(p, p->pev[2][0], B));
        if (k == K - 1) CU(ev_record_on(p, p->evb[0], B));
        if ((rc = Pass<T>::x_part(p, eoff(p->work, (long long)k * g.n0 * p->n1l * zk, p->esz), p->buf2, zk, k, k < K - 1 ? cap : 0, B))) return rc;
    }
    CU(ev_record_on(p, p->pev[2][1], B));
    CU(ev_record_on(p, p->evb[1], B));
    if (p2p && (rc = flags_signal(p, 0, p->epoch, B))) return rc;
    CU(ev_record_on(p, p->ev_join, B));
    CU(stream_wait(p, A, p->ev_join));
    CU(ev_record(p, p->ev[2]));
    CU(ev_record(p, p->ev[3]));
    p->timed = true;
    return 0;
}

// Stream-pipelined backward transform (P > 1): the mirror image of fwd_pipelined.  Send side (plan stream): the inverse X
// pass of z-part k, whose chunked store drops the x-planes of every destination straight into its receive buffer (P2P) or
// into the part-major send buffer followed by ncclAlltoAll of the part (NCCL).  Receive side (second stream): as soon as part k
// has arrived from every sender, the inverse Y pass of its columns (unpack folded into the load); the last part's Y pass
// completes every plane and runs fused with the inverse Z pass.  Receive layout of device p, part k:
// [sender q][x_l][y_l(q)][z'] at k * n0_l(p) * N1 * zk + q * n0_l(p) * yd * zk.
template <typename T> static int bwd_pipelined(dfft_plan p)
{
    const Geom& g = p->g;
    const int P = p->P, me = p->me, K = p->parts;
    const long long zk = g.n2 / K;
    const bool p2p = p->xmode == DFFT_EXCHANGE_P2P;
    const bool scale = (p->flags & DFFT_SCALE_BACKWARD) != 0;
    cudaStream_t A = p->stream, B = p->stream2, Cs = p->stream3;
    int rc = 0;
    struct Guard { dfft_plan p; ~Guard() { p->in_pipe = false; } } guard{p};
    p->in_pipe = true;
    int cap = 1;
    if (getenv("DFFT_PIPE_CAP")) cap = atoi(getenv("DFFT_PIPE_CAP"));
    if (p2p) {
        p->epoch++;
        if ((rc = flags_wait(p, 0, p->epoch - 1))) return rc;
    }
    CU(ev_record(p, p->pev[2][0]));
    for (int k = 0; k < K; k++) {
        void* base[DFFT_MAX_CHUNKS];
        for (int q = 0; q < P; q++)
            base[q] = p2p ? eoff(p->peer_work[q], ((long long)k * g.n1 + (long long)me * g.yd()) * g.n0l(q) * zk, p->esz)
                          : eoff(p->sendbuf, ((long long)k * P + q) * g.xd() * p->n1l * zk, p->esz);
        if ((rc = Pass<T>::xb_part(p, p->buf1, zk, k, base, k > 0 ? cap : 0))) return rc;
        if (p2p) {
            if (!p->done_ctr && (rc = flags_signal(p, 2 + k, p->epoch, A))) return rc;
        } else {
            const long long chunk = g.xd() * p->n1l * zk;
            CU(ev_record_on(p, p->ev_y[k], A));
            CU(stream_wait(p, Cs, p->ev_y[k]));
            if ((rc = nccl_exchange_part(p, eoff(p->sendbuf, (long long)k * P * chunk, p->esz), eoff(p->work, (long long)k * P * chunk, p->esz), chunk, Cs))) return rc;
            CU(ev_record_on(p, p->ev_a[k], Cs));
        }
    }
    CU(ev_record(p, p->pev[2][1]));
    CU(ev_record(p, p->ev[1]));
    for (int k = 0; k < K; k++) {
        if (p2p) { if ((rc = flags_wait(p, 2 + k, p->epoch, B))) return rc; }
        else CU(stream_wait(p, B, p->ev_a[k]));
        if (k == 0) CU(ev_record_on(p, p->pev[1][0], B));
        if (k == K - 1) CU(ev_record_on(p, p->evb[0], B));
        const void* rpart = eoff(p->work, (long long)k * p->n0l * g.n1 * zk, p->esz);
        if (k == K - 1 && p->fuse) rc = Pass<T>::yz_fused_last_part(p, rpart, p->buf2, zk, k, scale, B);
        else rc = Pass<T>::yinv_part(p, rpart, p->buf2, zk, k, k < K - 1 ? cap : 0, B);
        if (rc) return rc;
    }
    CU(ev_record_on(p, p->pev[1][1], B));
    if (!p->fuse) {
        // inverse Z pass of the whole slab on the receive stream (Pass::z_pass launches on the plan stream: join first)
        CU(ev_record_on(p, p->ev_join, B));
        CU(stream_wait(p, A, p->ev_join));
        if ((rc = Pass<T>::z_pass(p, p->buf2, p->buf2, scale, DFFT_BACKWARD))) return rc;
        CU(ev_record(p, p->evb[1]));
        CU(ev_record(p, p->pev[0][0])); CU(ev_record(p, p->pev[0][1]));
        if (p2p && (rc = flags_signal(p, 0, p->epoch, A))) return rc;
    } else {
        CU(ev_record_on(p, p->pev[0][0], B)); CU(ev_record_on(p, p->pev[0][1], B));
        CU(ev_record_on(p, p->evb[1], B));
        if (p2p && (rc = flags_signal(p, 0, p->epoch, B))) return rc;
        CU(ev_record_on(p, p->ev_join, B));
        CU(stream_wait(p, A, p->ev_join));
    }
    CU(ev_record(p, p->ev[2]));
    CU(ev_record(p, p->ev[3]));
    p->timed = true;
    return 0;
}

// ---- the non-pipelined slab schedule: forward half, X step, backward half -------------------------------------------------
// C2C / R2C forward = forward half + forward X, backward = backward X + backward half, convolve = forward half + fused X pass +
// backward half.  P2P gates and signals: the completion SIGNALS ride inside the pass kernels where the plan has done_ctr (their
// last CTA publishes the flags: fewer launches, DFFT_SIGNAL_KERNELS=1 restores the separate launches).  The GATES stay one-CTA
// kernels on purpose: a full-grid kernel that spins on a peer's flag holds every SM slot, and with two plans in flight per device
// (bench.py's e2e leg) device A can then wait for a kernel of device B that cannot start because B's SMs are held by a kernel
// waiting for A.  Flag words: ready[r] = e once receiver r has consumed its receive buffer of epoch e, arrive[s] = e once sender
// s has finished writing this device's receive buffer of epoch e.
static bool folds(dfft_plan p) { return p->P > 1 && p->xmode == DFFT_EXCHANGE_P2P && p->done_ctr != nullptr && !p->dry; }

// x-slab (bufferDev1) -> the receive buffer `work` [x][y_l][z'] of every device, epoch e: the Z step (fused with Y, or Z then Y),
// with the Y pass's store doing the pack (into `stage`, NCCL) or the all-to-all itself (into the peers' `work`, P2P)
template <typename T> static int fwd_half(dfft_plan p, unsigned long long e, bool fused, bool fused_tma)
{
    const Geom& g = p->g;
    const int P = p->P;
    const bool p2p = P > 1 && p->xmode == DFFT_EXCHANGE_P2P;
    void* zout = p2p ? p->stage : p->work;   // Z output; one device: Y runs in place in `work`
    void* ydst = P == 1 ? p->work : nullptr;
    const int ymode = P == 1 ? 0 : 1;
    void* base[DFFT_MAX_CHUNKS];
    if (P > 1)
        for (int q = 0; q < P; q++)
            base[q] = p2p ? eoff(p->peer_work[q], recv_off(g, p->me, q, DFFT_FORWARD), p->esz) : eoff(p->stage, send_off(g, p->me, q, DFFT_FORWARD), p->esz);
    Fold fy; fy.sig_which = 1; fy.sig_val = e; fy.ctr = 0;   // "arrived" from the Y pass's last CTA
    const Fold* fold = folds(p) ? &fy : nullptr;
    int rc;
    if (fused_tma) return Pass<T>::zy_fused_tma(p, p->buf1, p->work);
    if (fused) {
        if (p2p && (rc = flags_wait(p, 0, e - 1))) return rc;   // every receiver has consumed the previous epoch
        return Pass<T>::zy_fused(p, p->buf1, zout, ydst, ymode, base, false, fold, DFFT_FORWARD);
    }
    if (p->r2c) rc = Pass<T>::z_real(p, p->buf1, zout, false, DFFT_FORWARD);
    else rc = Pass<T>::z_pass(p, p->buf1, zout, false, DFFT_FORWARD);
    if (rc) return rc;
    if (p2p && (rc = flags_wait(p, 0, e - 1))) return rc;
    return Pass<T>::y_pass(p, zout, ydst, ymode, base, fold, DFFT_FORWARD);
}

// what follows the pass that sent epoch e: its "arrived" signal unless folded, event `sent`, the arrival wait (P2P) or the NCCL
// all-to-all of `stage` into `work`, event `arrived` (either event may be null)
static int deliver(dfft_plan p, unsigned long long e, int dir, cudaEvent_t sent, cudaEvent_t arrived)
{
    const bool p2p = p->P > 1 && p->xmode == DFFT_EXCHANGE_P2P;
    int rc;
    if (p2p && !folds(p) && (rc = flags_signal(p, 1, e))) return rc;
    if (sent) CU(ev_record(p, sent));
    if (p2p && (rc = flags_wait(p, 1, e))) return rc;   // exposed wait for the slowest sender
    if (p->P > 1 && !p2p && (rc = nccl_exchange(p, p->stage, p->work, dir))) return rc;
    if (arrived) CU(ev_record(p, arrived));
    return 0;
}

// receive buffer -> x-slab (bufferDev2), epoch e: Y from the chunks of `rbuf` (one device: from `src`) into `ybwd`, then Z (fused
// with Y, in place, or the real-data pass into bufferDev2), with "consumed" signalled once Y has read the receive buffer
template <typename T> static int bwd_half(dfft_plan p, unsigned long long e, bool fused, const void* src, void* rbuf, bool scale)
{
    const Geom& g = p->g;
    const int P = p->P;
    const bool p2p = P > 1 && p->xmode == DFFT_EXCHANGE_P2P;
    void* cb[DFFT_MAX_CHUNKS];
    if (P > 1)
        for (int q = 0; q < P; q++) cb[q] = eoff(rbuf, (long long)q * p->n0l * g.yd() * g.n2, p->esz);
    const void* ysrc = P == 1 ? src : nullptr;
    const int ymode = P == 1 ? 0 : 2;
    Fold fyz; fyz.sig_which = 0; fyz.sig_val = e; fyz.ctr = 1;   // the fused kernel is the last reader: its last CTA signals "consumed"
    const bool fold = fused && folds(p);
    int rc;
    if (fused) rc = Pass<T>::zy_fused(p, ysrc, p->ybwd, nullptr, ymode, cb, scale, fold ? &fyz : nullptr, DFFT_BACKWARD);
    else rc = Pass<T>::y_pass(p, ysrc, p->ybwd, ymode, cb, nullptr, DFFT_BACKWARD);
    if (rc) return rc;
    if (p2p && !fold && (rc = flags_signal(p, 0, e))) return rc;
    if (p->r2c) return Pass<T>::z_real(p, p->ybwd, p->buf2, scale, DFFT_BACKWARD);
    if (!fused) return Pass<T>::z_pass(p, p->buf2, p->buf2, scale, DFFT_BACKWARD);
    return 0;
}

// Overlapped forward (P2P): the whole transform in one kernel, t3 behind the per-part arrivals
template <typename T> static int execute_overlapped(dfft_plan p)
{
    const Geom& g = p->g;
    int rc;
    void* base[DFFT_MAX_CHUNKS];
    for (int q = 0; q < p->P; q++) base[q] = eoff(p->peer_work[q], recv_off(g, p->me, q, DFFT_FORWARD), p->esz);
    p->epoch++;
    if ((rc = flags_wait(p, 0, p->epoch - 1))) return rc;   // every receiver has consumed the previous epoch
    if ((rc = Pass<T>::fwd_overlapped(p, base))) return rc;
    CU(ev_record(p, p->ev[1]));
    CU(ev_record(p, p->ev[2]));
    if ((rc = flags_signal(p, 0, p->epoch))) return rc;
    CU(ev_record(p, p->ev[3]));
    p->timed = true;
    return 0;
}

// Convolve plans: out = IFFT3(m .* FFT3(in)), never writing bufferDev1.  The forward half is the C2C (R2C) forward schedule up to
// the arrival of the receive buffer [x][y_l][z'], the fused X pass (fft_conv_kernel) replaces the forward X pass, the multiply and
// the backward X pass, and the backward half is the C2C (C2R) backward schedule from the exchange on.  Buffers:
//   P = 1 : work (forward t0 out, fused X pass in place, backward t0 in); bufferDev2 (= out) gets the result
//   NCCL  : work = both exchanges' receive buffer, mid = forward send buffer, fused X pass output (already grouped by destination:
//           it is the backward send buffer) and, R2C, the backward Y output
//   P2P   : work = forward receive buffer, work2 = backward receive buffer (the fused X pass stores into the peers' work2),
//           mid = forward Z output and, R2C, the backward Y output
// Epochs (P2P): execute k uses e1 = 2k+1 for the forward exchange and e2 = 2k+2 for the backward one; arrive[s] takes e1 then e2
// from sender s, ready[r] takes e2 once receiver r's backward Y pass has read its work2.  No device writes a peer buffer before
// the owner has finished reading that buffer's previous contents:
//   * the forward Y stores into peer r's work wait for ready[r] >= e1 - 1 (= e2 of the previous execute): r's backward Y pass of
//     the previous execute is done, and with it r's fused X pass, the only reader of r's work;
//   * the fused X pass stores into peer r's work2 behind the same gate (it runs later on the same stream): r's backward Y pass of
//     the previous execute, the only reader of r's work2, is done;
//   * the waits are >= tests on monotonic words: the previous execute's e2 (= e1 - 1) never satisfies the wait for e1, and a sender
//     publishes e2 only from its fused X pass, after every store of its forward Y pass.
template <typename T> static int execute_slabs(dfft_plan p, const void* mult)
{
    const Geom& g = p->g;
    const int P = p->P, me = p->me;
    const bool p2p = P > 1 && p->xmode == DFFT_EXCHANGE_P2P;
    int rc;
    p->launches = 0;
    CU(ev_record(p, p->ev[0]));
    if (p->pipe) return p->direction == DFFT_FORWARD ? fwd_pipelined<T>(p) : bwd_pipelined<T>(p);
    if (p->overlap) return execute_overlapped<T>(p);
    unsigned long long e1 = 0, e2 = 0;   // epochs of the forward and the backward exchange (one of them for C2C / R2C)
    if (p2p) {
        e1 = ++p->epoch;
        e2 = p->conv ? ++p->epoch : e1;
    }
    void* base[DFFT_MAX_CHUNKS];
    if (p->conv) {
        if ((rc = fwd_half<T>(p, e1, p->conv_fuse[0], p->conv_fuse_tma))) return rc;
        if ((rc = deliver(p, e1, DFFT_FORWARD, nullptr, p->ev[1]))) return rc;
        Fold fc; fc.sig_which = 1; fc.sig_val = e2; fc.ctr = 1;
        if (P == 1) rc = Pass<T>::x_conv(p, p->work, p->work, nullptr, mult, nullptr);
        else if (p2p) {
            for (int q = 0; q < P; q++) base[q] = eoff(p->peer_work2[q], recv_off(g, me, q, DFFT_BACKWARD), p->esz);
            rc = Pass<T>::x_conv(p, p->work, nullptr, base, mult, folds(p) ? &fc : nullptr);
        } else rc = Pass<T>::x_conv(p, p->work, p->stage, nullptr, mult, nullptr);   // [x][y_l][z'] is grouped by destination
        if (rc) return rc;
        if ((rc = deliver(p, e2, DFFT_BACKWARD, p->ev[2], nullptr))) return rc;
        if ((rc = bwd_half<T>(p, e2, p->conv_fuse[1], p->work, p2p ? p->work2 : p->work, false))) return rc;
    } else if (p->direction == DFFT_FORWARD) {
        if ((rc = fwd_half<T>(p, e1, p->fuse, p->fuse_tma))) return rc;
        if ((rc = deliver(p, e1, DFFT_FORWARD, p->ev[1], p->ev[2]))) return rc;
        Fold fx; fx.sig_which = 0; fx.sig_val = e1; fx.ctr = 1;   // "consumed" from the X pass's last CTA (not on the TMA kernel)
        const bool foldx = folds(p) && Pass<T>::x_fwd_folds(p);
        if (p->natural) rc = Pass<T>::x_natural(p, p->work, p->buf2);
        else rc = Pass<T>::x_fwd(p, p->work, p->buf2, foldx ? &fx : nullptr);
        if (rc) return rc;
        if (p2p && !foldx && (rc = flags_signal(p, 0, e1))) return rc;
    } else {
        Fold fxb; fxb.sig_which = 1; fxb.sig_val = e1; fxb.ctr = 0;
        if (P == 1) rc = p->natural ? Pass<T>::x_natural(p, p->buf1, p->ybwd) : Pass<T>::x_bwd(p, p->buf1, p->ybwd, nullptr);
        else if (p2p) {
            if ((rc = flags_wait(p, 0, e1 - 1))) return rc;
            for (int q = 0; q < P; q++) base[q] = eoff(p->peer_work[q], recv_off(g, me, q, DFFT_BACKWARD), p->esz);
            rc = Pass<T>::x_bwd(p, p->buf1, nullptr, base, folds(p) ? &fxb : nullptr);
        } else rc = Pass<T>::x_bwd(p, p->buf1, p->stage, nullptr);
        if (rc) return rc;
        if ((rc = deliver(p, e1, DFFT_BACKWARD, p->ev[1], p->ev[2]))) return rc;
        if ((rc = bwd_half<T>(p, e1, p->fuse, p->ybwd, p->work, (p->flags & DFFT_SCALE_BACKWARD) != 0))) return rc;
    }
    CU(ev_record(p, p->ev[3]));
    p->timed = true;
    return 0;
}

// reference-like stage-by-stage execution (api.cpp:181-214 with its device-wide syncs)
template <typename T> static int execute_stage(dfft_plan p, int stage)
{
    const Geom& g = p->g;
    const int P = p->P, me = p->me, dir = p->direction;
    int rc = 0;
    // map "k-th executed stage" to the reference stage id
    const int sid = dir == DFFT_FORWARD ? stage : 3 - stage;
    if (sid == 0) {          // fftZY
        void* buf = dir == DFFT_FORWARD ? p->buf1 : p->buf2;
        if (dir == DFFT_FORWARD) {
            if ((rc = Pass<T>::z_pass(p, buf, buf, false, dir))) return rc;
            if ((rc = Pass<T>::y_pass(p, buf, buf, 0, nullptr, nullptr, dir))) return rc;
        } else {
            if ((rc = Pass<T>::y_pass(p, buf, buf, 0, nullptr, nullptr, dir))) return rc;
            if ((rc = Pass<T>::z_pass(p, buf, buf, (p->flags & DFFT_SCALE_BACKWARD) != 0, dir))) return rc;
        }
    } else if (sid == 1) {   // localTransposeUneven
        cudaError_t e = launch_pack_rows(p->buf1, p->buf2, (int)p->esz, p->n0l, g.n1, g.n2, P, dir == DFFT_FORWARD, p->sms, p->stream);
        if (e != cudaSuccess) return fail(DFFT_ECUDA, "pack launch failed: %s", cudaGetErrorString(e));
        p->launches++;
    } else if (sid == 2) {   // slabAlltoall
        if (P > 1) {
            CU(cudaStreamSynchronize(p->stream));
            p->comm->host_barrier(me);   // every sender's buf2 is packed, every receiver's buf1 is free
            for (int q = 0; q < P; q++) {
                CU(cudaMemcpyAsync(eoff(p->peer_buf1[q], recv_off(g, me, q, dir), p->esz), eoff(p->buf2, send_off(g, me, q, dir), p->esz),
                                   (size_t)xchg_count(g, me, q, dir) * p->esz, cudaMemcpyDefault, p->stream));
                p->launches++;
            }
            CU(cudaStreamSynchronize(p->stream));
            p->comm->host_barrier(me);
        } else {
            CU(cudaMemcpyAsync(p->buf1, p->buf2, (size_t)p->in_count * p->esz, cudaMemcpyDeviceToDevice, p->stream));
            p->launches++;
        }
    } else {                 // fftX
        if (dir == DFFT_FORWARD) rc = Pass<T>::x_fwd(p, p->buf1, p->buf2);
        else rc = Pass<T>::x_bwd(p, p->buf1, p->buf2, nullptr);
        if (rc) return rc;
    }
    CU(cudaStreamSynchronize(p->stream));
    return 0;
}

extern "C" int dfft_execute_stage(dfft_plan p, int stage)
{
    if (p && p->conv) return fail(DFFT_EINVAL, "dfft_execute_stage: a convolve plan runs with dfft_execute_convolve");
    if (p && p->r2c) return fail(DFFT_EUNSUPPORTED, "dfft_execute_stage: R2C / C2R plans have no stage-by-stage mode");
    if (!p || stage < 0 || stage > 3 || p->dry) return fail(DFFT_EINVAL, "dfft_execute_stage: bad arguments");
    if (p->xmode != DFFT_EXCHANGE_STAGED) return fail(DFFT_EINVAL, "dfft_execute_stage needs a plan created with DFFT_EXCHANGE_STAGED");
    CU(cudaSetDevice(p->device));
    return p->prec == DFFT_DOUBLE ? execute_stage<double>(p, stage) : execute_stage<float>(p, stage);
}

extern "C" int dfft_execute(dfft_plan p)
{
    if (!p) return fail(DFFT_EINVAL, "null plan");
    if (p->conv) return fail(DFFT_EINVAL, "dfft_execute: a convolve plan runs with dfft_execute_convolve");
    if (p->dry) p->ops.clear();
    else CU(cudaSetDevice(p->device));
    if (p->xmode == DFFT_EXCHANGE_STAGED) {
        p->launches = 0;
        for (int s = 0; s < 4; s++) {
            CU(ev_record(p, p->ev[s]));
            int rc = p->prec == DFFT_DOUBLE ? execute_stage<double>(p, s) : execute_stage<float>(p, s);
            if (rc) return rc;
        }
        CU(ev_record(p, p->ev[4]));
        p->timed = true;
        return 0;
    }
    return p->prec == DFFT_DOUBLE ? execute_slabs<double>(p, nullptr) : execute_slabs<float>(p, nullptr);
}

extern "C" int dfft_execute_convolve(dfft_plan p, const void* multiplier)
{
    if (!p) return fail(DFFT_EINVAL, "null plan");
    if (!p->conv) return fail(DFFT_EINVAL, "dfft_execute_convolve needs a plan from dfft_plan_convolve_c2c_3d / dfft_plan_convolve_r2c_3d");
    if (!multiplier) return fail(DFFT_EINVAL, "dfft_execute_convolve: null multiplier");
    if ((uintptr_t)multiplier % p->esz) return fail(DFFT_EINVAL, "dfft_execute_convolve: the multiplier is not aligned to its complex element size (%zu bytes)", p->esz);
    if (p->dry) p->ops.clear();
    else CU(cudaSetDevice(p->device));
    return p->prec == DFFT_DOUBLE ? execute_slabs<double>(p, multiplier) : execute_slabs<float>(p, multiplier);
}

extern "C" int dfft_synchronize(dfft_plan p)
{
    if (!p) return fail(DFFT_EINVAL, "null plan");
    if (p->dry) return 0;
    CU(cudaSetDevice(p->device));
    CU(cudaStreamSynchronize(p->stream));
    return 0;
}

extern "C" int dfft_get_timings(dfft_plan p, double t[5])
{
    if (!p || !t) return fail(DFFT_EINVAL, "bad arguments");
    if (!p->timed || p->dry) return fail(DFFT_EINVAL, "no execute to time yet");
    CU(cudaSetDevice(p->device));
    CU(cudaStreamSynchronize(p->stream));
    float ms[4] = {0, 0, 0, 0};
    if (p->xmode == DFFT_EXCHANGE_STAGED) {
        for (int s = 0; s < 4; s++) CU(cudaEventElapsedTime(&ms[s], p->ev[s], p->ev[s + 1]));
        if (p->direction == DFFT_BACKWARD) { std::swap(ms[0], ms[3]); std::swap(ms[1], ms[2]); }
        for (int s = 0; s < 4; s++) t[s] = ms[s];
    } else if (p->conv) {
        // convolve: t0 = forward half (its t0 and exchange), t3 = fused X pass, t2 = backward half (its exchange and t0)
        float a, b, c;
        CU(cudaEventElapsedTime(&a, p->ev[0], p->ev[1]));
        CU(cudaEventElapsedTime(&b, p->ev[1], p->ev[2]));
        CU(cudaEventElapsedTime(&c, p->ev[2], p->ev[3]));
        t[0] = a; t[1] = 0; t[2] = c; t[3] = b;
    } else if (p->pipe) {
        // send side [start, last part issued] = t0 (+t1, + the sends); exposed exchange = from there until the last part has
        // arrived from every sender; t3 = the X pass of the last part (the earlier parts ran under t0)
        float a, b, c;
        CU(cudaEventElapsedTime(&a, p->ev[0], p->ev[1]));
        CU(cudaEventElapsedTime(&b, p->ev[1], p->evb[0]));
        CU(cudaEventElapsedTime(&c, p->evb[0], p->evb[1]));
        if (b < 0) { c += b; b = 0; }
        if (p->direction == DFFT_FORWARD) { t[0] = a; t[1] = 0; t[2] = b; t[3] = c; }
        else { t[3] = a; t[2] = b; t[1] = 0; t[0] = c; }   // backward: the send side is t3 (inverse X), the receive tail t0
    } else {
        float a, b, c;
        CU(cudaEventElapsedTime(&a, p->ev[0], p->ev[1]));
        CU(cudaEventElapsedTime(&b, p->ev[1], p->ev[2]));
        CU(cudaEventElapsedTime(&c, p->ev[2], p->ev[3]));
        if (p->direction == DFFT_FORWARD) { t[0] = a; t[1] = 0; t[2] = b; t[3] = c; }
        else { t[3] = a; t[2] = b; t[1] = 0; t[0] = c; }
    }
    t[4] = t[0] + t[1] + t[2] + t[3];
    return 0;
}

extern "C" int dfft_get_pass_timings(dfft_plan p, double t[3])
{
    if (!p || !t) return fail(DFFT_EINVAL, "bad arguments");
    if (!p->timed || p->dry) return fail(DFFT_EINVAL, "no execute to time yet");
    CU(cudaSetDevice(p->device));
    CU(cudaStreamSynchronize(p->stream));
    for (int a = 0; a < 3; a++) {
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, p->pev[a][0], p->pev[a][1]));
        t[a] = ms;
    }
    return 0;
}

extern "C" int dfft_execute_host_async(dfft_plan p, const void* host_in, void* host_out)
{
    if (!p || !host_in || !host_out || p->dry) return fail(DFFT_EINVAL, "bad arguments");
    if (p->conv) return fail(DFFT_EINVAL, "dfft_execute_host: a convolve plan runs with dfft_execute_convolve");
    CU(cudaSetDevice(p->device));
    CU(cudaMemcpyAsync(p->buf1, host_in, (size_t)p->in_count * p->in_esz, cudaMemcpyHostToDevice, p->stream));
    int rc = dfft_execute(p);
    if (rc) return rc;
    CU(cudaMemcpyAsync(host_out, p->buf2, (size_t)p->out_count * p->out_esz, cudaMemcpyDeviceToHost, p->stream));
    return 0;
}

extern "C" int dfft_execute_host(dfft_plan p, const void* host_in, void* host_out)
{
    int rc = dfft_execute_host_async(p, host_in, host_out);
    if (rc) return rc;
    CU(cudaStreamSynchronize(p->stream));
    return 0;
}

extern "C" int dfft_plan_buffers(dfft_plan p, void** b1, void** b2)
{
    if (!p) return fail(DFFT_EINVAL, "null plan");
    if (b1) *b1 = p->buf1;
    if (b2) *b2 = p->buf2;
    return 0;
}
extern "C" int dfft_plan_counts(dfft_plan p, long long* ic, long long* oc, long long* mc)
{
    if (!p) return fail(DFFT_EINVAL, "null plan");
    if (ic) *ic = p->in_count;
    if (oc) *oc = p->out_count;
    if (mc) *mc = p->max_count;
    return 0;
}
/* test hook: JSON array of the passes the last dfft_execute of a DFFT_DRY_RUN plan recorded; returns the length needed */
extern "C" long long dfft_debug_plan_ops(dfft_plan p, char* buf, long long cap)
{
    if (!p) return -1;
    return ops_json(p->ops, buf, cap);
}

static_assert(sizeof(((dfft_debug_chunks*)nullptr)->cptr) / sizeof(void*) == DFFT_MAX_CHUNKS, "dfft_debug_chunks mirrors ChunkTab");

// one record of dfft_debug_launch_op as the kernel's TileArgs; the checks every kind shares.  want_ci / want_co: the kind loads /
// stores through a chunk table (which must then be given, and must not be otherwise)
template <typename T>
static int replay_args(const char* name, const dfft_debug_op* r, const SizeEntry* e, int C, bool want_ci, bool want_co, TileArgs<T>& a)
{
    if (r->C != C) return fail(DFFT_EINVAL, "dfft_debug_launch_op: %s record of N=%d has C=%d, the entry's configuration has %d", name, r->N, r->C, C);
    if (r->G < 1 || r->ntiles < 0 || r->ntiles % r->G || r->W <= (long long)(r->G - 1) * C || r->W > (long long)r->G * C)
        return fail(DFFT_EINVAL, "dfft_debug_launch_op: %s record with inconsistent G=%d, W=%d, ntiles=%lld (C=%d)", name, r->G, r->W, r->ntiles, C);
    const dfft_debug_chunks* side[2] = {&r->ci, &r->co};
    const bool want[2] = {want_ci, want_co};
    ChunkTab* tab[2] = {&a.ci, &a.co};
    for (int s = 0; s < 2; s++) {
        const dfft_debug_chunks& ch = *side[s];
        if (!want[s]) {
            if (ch.nchunks != 0) return fail(DFFT_EINVAL, "dfft_debug_launch_op: %s takes no chunk table on its %s side", name, s ? "store" : "load");
            continue;
        }
        if (ch.nchunks < 1 || ch.nchunks > DFFT_MAX_CHUNKS || ch.ediv < 1)
            return fail(DFFT_EINVAL, "dfft_debug_launch_op: %s needs a chunk table on its %s side", name, s ? "store" : "load");
        for (int q = 0; q < ch.nchunks; q++) {
            if (!ch.cptr[q]) return fail(DFFT_EINVAL, "dfft_debug_launch_op: %s chunk %d has a null pointer", name, q);
            tab[s]->cptr[q] = ch.cptr[q];
            tab[s]->SAq[q] = ch.SAq[q];
        }
        tab[s]->ediv = ch.ediv;
        tab[s]->nchunks = ch.nchunks;
    }
    if ((!want_ci && !r->in) || (!want_co && !r->out)) return fail(DFFT_EINVAL, "dfft_debug_launch_op: %s record with a null buffer", name);
    a.in = (const cx<T>*)r->in; a.out = (cx<T>*)r->out;
    a.ia = Affine{r->ia[0], r->ia[1], r->ia[2], r->ia[3]};
    a.oa = Affine{r->oa[0], r->oa[1], r->oa[2], r->oa[3]};
    a.ntiles = r->ntiles; a.G = r->G; a.W = r->W;
    a.inv = r->inv ? 1 : 0; a.do_scale = r->do_scale ? 1 : 0; a.scale = (T)r->scale;
    a.tw_n = r->tw_n;
    a.gen = e->gen;
    return 0;
}

template <typename T>
static int replay_op(const char* op, const dfft_debug_op* r, const char* op2, const dfft_debug_op* r2, int precision)
{
    int sms = 132, dev = 0;
    CU(cudaGetDevice(&dev));
    CU(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const SizeEntry* e = find_size_entry(r->N, precision);
    if (!e) return fail(DFFT_EINVAL, "dfft_debug_launch_op: no kernel entry of length %d", r->N);
    const bool fz = !strcmp(op, "fusedZ"), fy = !strcmp(op, "fusedY");
    std::vector<void*> owned;   // twiddle tables and fused controls of this launch
    auto release = [&](int rc) {
        for (void* q : owned) cudaFree(q);
        return rc;
    };
#define CUR(x)                                                                                        \
    do {                                                                                              \
        cudaError_t e_ = (x);                                                                         \
        if (e_ != cudaSuccess) return release(fail(DFFT_ECUDA, "%s:%d CUDA call '%s' failed: %s", __FILE__, __LINE__, #x, cudaGetErrorString(e_))); \
    } while (0)
    auto lut = [&](int kind, const cx<T>** out) {
        void* d = nullptr;
        const cudaError_t err = upload_lut_kind<T>(&d, e, kind);
        if (d) owned.push_back(d);
        *out = (const cx<T>*)d;
        return err;
    };
    cudaError_t err;
    if (fz || fy) {
        // the two roles of a t0 kernel, records in their recorded order: forward fusedZ + fusedY (FK_ZY_CO with the chunked
        // store), backward fusedY + fusedZ (FK_YZ_CI with the chunked load)
        const char* other = fz ? "fusedY" : "fusedZ";
        if (!r2 || !op2 || strcmp(op2, other)) return fail(DFFT_EINVAL, "dfft_debug_launch_op: %s needs its %s record", op, other);
        if (r2->N != r->N) return fail(DFFT_EINVAL, "dfft_debug_launch_op: the fused roles have lengths %d and %d", r->N, r2->N);
        const dfft_debug_op& zr = fz ? *r : *r2;
        const dfft_debug_op& yr = fz ? *r2 : *r;
        const bool chunked = fz ? yr.co.nchunks != 0 : yr.ci.nchunks != 0;
        const int kind = fz ? (chunked ? FK_ZY_CO : FK_ZY) : (chunked ? FK_YZ_CI : FK_YZ);
        const int CZ = kind == FK_ZY_CO ? e->f_zCp : e->f_zC, CY = kind == FK_ZY_CO ? e->p_C : e->s_C;
        if (!e->fused[kind]) return fail(DFFT_EUNSUPPORTED, "dfft_debug_launch_op: length %d has no fused kernel of kind %d", r->N, kind);
        TileArgs<T> z{}, y{};
        int rc = replay_args<T>("fusedZ", &zr, e, CZ, false, false, z);
        if (!rc) rc = replay_args<T>("fusedY", &yr, e, CY, !fz && chunked, fz && chunked, y);
        if (rc) return rc;
        if (z.ntiles / z.G != y.ntiles / y.G) return fail(DFFT_EINVAL, "dfft_debug_launch_op: the fused roles cover different planes");
        CUR(lut(PK_Z, &z.lut));
        CUR(lut(PK_Y, &y.lut));
        // as fused_ctl does for the first execute of a plan: zeroed plane counters and ticket words, role A done at GA
        FusedCtl c{};
        c.planes = z.ntiles / z.G;
        c.GA = fz ? z.G : y.G; c.GB = fz ? y.G : z.G;
        c.target = (unsigned long long)c.GA;
        c.lag = 0;
        CUR(cudaMalloc((void**)&c.plane_done, (size_t)std::max<long long>(c.planes, 1) * sizeof(unsigned long long)));
        owned.push_back(c.plane_done);
        CUR(cudaMemset(c.plane_done, 0, (size_t)std::max<long long>(c.planes, 1) * sizeof(unsigned long long)));
        CUR(cudaMalloc((void**)&c.ticket, 4 * sizeof(unsigned int)));
        owned.push_back(c.ticket);
        CUR(cudaMemset(c.ticket, 0, 4 * sizeof(unsigned int)));
        err = fz ? e->fused[kind](&z, &y, &c, sms, nullptr) : e->fused[kind](&y, &z, &c, sms, nullptr);
    } else {
        int kind = -1;
        for (int k = 0; k < PK_COUNT; k++)
            if (!strcmp(op, kPassNames[k])) kind = k;
        if (kind < 0 || kind == PK_Z_R2C || kind == PK_Z_C2R || kind >= PK_PLANE)
            return fail(DFFT_EINVAL, "dfft_debug_launch_op: '%s' is not a record this hook launches", op);
        if (!e->launch[kind]) return fail(DFFT_EUNSUPPORTED, "dfft_debug_launch_op: length %d has no %s kernel", r->N, op);
        if (r2 || op2) return fail(DFFT_EINVAL, "dfft_debug_launch_op: %s is one record", op);
        const bool conv = kind == PK_XCONV || kind == PK_XCONV_CO;
        if (conv && !r->mult) return fail(DFFT_EINVAL, "dfft_debug_launch_op: %s record with a null multiplier", op);
        ConvArgs<T> cv{};
        TileArgs<T>& a = cv.t;
        const int rc = replay_args<T>(op, r, e, kind_C(e, kind), kind == PK_Y_CI, kind == PK_Y_CO || kind == PK_XB_CO || kind == PK_XCONV_CO, a);
        if (rc) return rc;
        CUR(lut(kind, &a.lut));
        cv.mult = (const cx<T>*)r->mult;
        err = e->launch[kind](conv ? (const void*)&cv : (const void*)&a, sms, nullptr);
    }
    if (err != cudaSuccess) cudaGetLastError();   // a refused launch must not be reported again by the next one
    CUR(err);
    CUR(cudaStreamSynchronize(nullptr));
#undef CUR
    return release(0);
}

/* test hook: launch one record of a DFFT_DRY_RUN plan (see dfft.h) */
extern "C" int dfft_debug_launch_op(const char* op, const dfft_debug_op* rec, const char* second_op, const dfft_debug_op* second, int precision)
{
    if (!op || !rec) return fail(DFFT_EINVAL, "dfft_debug_launch_op: null record");
    if (precision != DFFT_DOUBLE && precision != DFFT_FLOAT) return fail(DFFT_EINVAL, "dfft_debug_launch_op: bad precision");
    if (!strcmp(op, "ovlZ") || !strcmp(op, "ovlY") || !strcmp(op, "ovlX"))
        return fail(DFFT_EINVAL, "dfft_debug_launch_op: the single-kernel forward (%s) waits on its peers' arrival flags", op);
    return precision == DFFT_DOUBLE ? replay_op<double>(op, rec, second_op, second, precision) : replay_op<float>(op, rec, second_op, second, precision);
}

extern "C" int dfft_plan_launches(dfft_plan p) { return p ? p->launches : 0; }
extern "C" int dfft_plan_exchange(dfft_plan p) { return p ? p->xmode : 0; }
/* bit 0 / 1 / 2: the un-chunked Z / Y / X pass of this plan runs on the TMA-pipelined kernel (fft_tma.cuh) */
extern "C" int dfft_plan_tma_mask(dfft_plan p)
{
    if (!p) return 0;
    const Geom& g = p->g;
    return (tma_ok(p, TMA_Z, p->n0l * g.n1) ? 1 : 0) | (tma_ok(p, TMA_Y, g.n2) ? 2 : 0) |
           (tma_ok(p, p->direction == DFFT_FORWARD ? TMA_XF : TMA_XB, g.n2) ? 4 : 0);
}
/* developer hook (DFFT_DEBUG_TIMELINE=1, single-kernel forward path): device-side timeline of the last execute, microseconds
 * relative to the kernel's start: [0] end of phase 0, [1] first X tile, [2] kernel end, [3..5] mean us per Z / Y / X tile,
 * [6..8] tile counts, [9] mean X-side wait per CTA, [10] max wait */
extern "C" int dfft_debug_timeline(dfft_plan p, double out[11])
{
    if (!p || !p->dbg || !out) return fail(DFFT_EINVAL, "no timeline recorded (set DFFT_DEBUG_TIMELINE=1 and use DFFT_OVERLAP_X)");
    CU(cudaSetDevice(p->device));
    CU(cudaStreamSynchronize(p->stream));
    unsigned long long h[16];
    CU(cudaMemcpy(h, p->dbg, sizeof(h), cudaMemcpyDeviceToHost));
    const double t0 = (double)h[0];
    out[0] = ((double)h[4] - t0) * 1e-3; out[1] = ((double)h[1] - t0) * 1e-3; out[2] = ((double)h[5] - t0) * 1e-3;
    for (int r = 0; r < 3; r++) { out[3 + r] = h[9 + r] ? (double)h[6 + r] / (double)h[9 + r] * 1e-3 : 0; out[6 + r] = (double)h[9 + r]; }
    const double ctas = (double)p->sms * 2;
    out[9] = (double)h[12] / ctas * 1e-3; out[10] = (double)h[13] * 1e-3;
    return 0;
}
extern "C" int dfft_plan_pipeline_parts(dfft_plan p) { return p && p->pipe ? p->parts : 0; }
/* 1: the parts run as a chain of two-role kernels on one stream (fft_fused_yx_kernel), 0: two streams / not pipelined */
extern "C" int dfft_plan_pipeline_chain(dfft_plan p) { return p && p->pipe && p->pipe_fyx ? 1 : 0; }
extern "C" int dfft_plan_fused(dfft_plan p) { return p && p->fuse && p->xmode != DFFT_EXCHANGE_STAGED ? (p->overlap ? 2 : 1) : 0; }
extern "C" void* dfft_plan_stream(dfft_plan p) { return p ? (void*)p->stream : nullptr; }

// ------------------------------------------------------------------------------------------------
// batched local transforms: plan / launch / delete, the templateFFT engine surface
// (3dmpifft_opt/include/templateFFT.h:361-365 initializeFFT / launchFFTKernel / deleteFFT)
// ------------------------------------------------------------------------------------------------
enum { LB_IN = 0, LB_TEMP = 1, LB_OUT = 2 };
struct LinePass {
    const SizeEntry* e = nullptr;
    int kind = PK_Z;             // a PassKind
    void* lut = nullptr;
    Affine ia{}, oa{};           // plane kinds, for the records: plane (image), 0, row and point strides
    int G = 0, W = 0;
    long long ntiles = 0;        // plane kinds: planes (images)
    long long tw_n = 0;          // four-step twiddle modulus (PK_XF_TW)
    int src = LB_IN, dst = LB_IN;   // LB_IN (the caller's data / a real or convolve plan's `in`), LB_TEMP (the plan's temporary), LB_OUT
    long long ld_in = 0, ld_out = 0;   // PK_Z_R2C / PK_Z_C2R / PK_LINE_CONV_R2C: distance between the two lines of a pair (RealZArgs), each side's elements
    bool inv = false;            // the inverse transform
};
// which execute runs a plan: dfft_lines_execute, dfft_lines_execute_real or dfft_lines_execute_convolve
enum LinesForm { LF_COMPLEX, LF_REAL, LF_CONV };
struct dfft_lines_plan_s {
    int prec = 0, device = 0, sms = 132;
    LinesForm form = LF_COMPLEX;
    bool real = false;           // convolve: real in / real out (dfft_lines_execute_convolve's element size and buffer extents)
    // the passes of one execute in order, [0] forward, [1] backward (a convolve plan has one list, [0]).  The create path launches
    // them and the dfft_debug_lines*_ops hooks record them, both through line_pass
    LinePass run[2][5];
    int nrun[2] = {0, 0};
    void* temp = nullptr;
    size_t temp_bytes = 0;       // the temporary a plan needs, allocated by lines_create
    struct Lut { const SizeEntry* e; int kind; void* d; };
    std::vector<Lut> luts;       // twiddle tables, one per (entry, schedule), shared by the passes that run it
    long long rcount = 0, ccount = 0;   // reals and complex elements of the caller's real / complex buffer
    long long batch = 0, mvol = 0;   // convolve: volumes (images); complex elements of one volume's (image's) multiplier
    double scale = 0;                // DFFT_SCALE_BACKWARD: 1 / (elements of a volume or image), folded into the multiply; 0 = unnormalised
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr};
};

static bool bad_precision(int precision) { return precision != DFFT_DOUBLE && precision != DFFT_FLOAT; }

// a * b * c < 2^31 (the kernels' 32-bit row counts TileArgs::W / G), without overflow for any non-negative arguments
static bool fits_int(long long a, long long b = 1, long long c = 1)
{
    return (__int128)a * b * c <= 0x7fffffff;
}

// the plain pass kind whose tile size (kind_C) and twiddle schedule (upload_lut_kind) a lines pass has: the real kernels run the
// contiguous configuration, the column convolve the strided one, the plane kernels the contiguous schedule and the line convolve
// kernels the contiguous configuration
static int plain_kind(int kind)
{
    return kind == PK_XCONV ? PK_Y : (kind == PK_Z_R2C || kind == PK_Z_C2R || kind >= PK_PLANE) ? PK_Z : kind;
}

// columns that touch no element twice: the (extent, stride) pairs (inner, 1), (n, stride) and (mats, outer_dist), sorted by
// stride, each have a stride at least the span of the ones before (the usual test for a non-overlapping strided tensor; pairs of
// extent 1 take no part, so a single matrix ignores outer_dist).  A negative outer_dist over two or more matrices fails it.
static bool columns_disjoint(int n, long long stride, long long inner, long long mats, long long outer_dist)
{
    struct Dim { long long extent, stride; } d[3] = {{inner, 1}, {n, stride}, {mats, outer_dist}};
    std::sort(d, d + 3, [](const Dim& a, const Dim& b) { return a.stride < b.stride; });
    __int128 span = 1;
    for (const Dim& x : d) {
        if (x.extent <= 1) continue;
        if (x.stride < span) return false;
        span += (__int128)(x.extent - 1) * x.stride;
    }
    return true;
}

// one pass over `nlines` lines of n points: densely packed contiguous lines (stride 1, PK_Z) or disjoint columns (inner_dist 1,
// PK_Y).  The pass's row or column count W is a 32-bit kernel argument
static int make_line_pass(LinePass& lp, int n, long long stride, long long nlines, long long inner, long long inner_dist, long long outer_dist,
                          int precision)
{
    const SizeEntry* e = find_size_entry(n, precision);
    if (!e) return fail(DFFT_EUNSUPPORTED, "unsupported length %d", n);
    lp.e = e;
    if (stride == 1) {
        if (inner_dist != n || (inner != nlines && outer_dist != inner * n)) return fail(DFFT_EUNSUPPORTED, "contiguous lines must be densely packed");
        if (!fits_int(nlines)) return fail(DFFT_EUNSUPPORTED, "%lld rows: at most 2^31 - 1 per plan", nlines);
        const int C = e->z_C;
        lp.G = (int)cdiv(nlines, C); lp.W = (int)nlines; lp.ntiles = lp.G;
        lp.ia = Affine{0, (long long)C * n, n, 1};
        lp.oa = lp.ia;
        lp.kind = PK_Z;
    } else {
        if (inner_dist != 1 || inner < 1 || nlines % inner) return fail(DFFT_EUNSUPPORTED, "strided lines must be columns (inner_dist == 1)");
        if (!fits_int(inner)) return fail(DFFT_EUNSUPPORTED, "%lld columns: at most 2^31 - 1 per pass", inner);
        if (!columns_disjoint(n, stride, inner, nlines / inner, outer_dist))
            return fail(DFFT_EINVAL, "columns overlap: %lld columns, n = %d, stride %lld, outer_dist %lld", inner, n, stride, outer_dist);
        const int C = e->s_C;
        lp.G = (int)cdiv(inner, C); lp.W = (int)inner; lp.ntiles = (nlines / inner) * lp.G;
        lp.ia = Affine{outer_dist, C, 1, stride};
        lp.oa = lp.ia;
        lp.kind = PK_Y;
    }
    return 0;
}

// complex plans: the backward list is the forward list inverted, in reverse order (ordered, four-step: in the same order)
static int complex_lists(dfft_lines_plan p, int n, bool ordered)
{
    p->nrun[0] = p->nrun[1] = n;
    for (int k = 0; k < n; k++) {
        p->run[1][k] = p->run[0][ordered ? k : n - 1 - k];
        p->run[1][k].inv = true;
    }
    return 0;
}

// Long contiguous lines (beyond one shared-memory line): four-step decomposition n = n1 * n2 in two passes,
//   A: view the line as [n1][n2]; FFT along n1 (stride n2), multiply by W_n^(n2*k1), store transposed -> temp [n2][k1]
//   B: FFT along n2 (stride n1) of temp, stored to the caller's buffer at [k2][k1] = natural order X[k1 + n1*k2]
// -- what the reference does with its multi-upload axes and reorderFourStep = 1 (templateFFT.cpp:4007-4106, 5951).
// Validated against numpy (tests/test_gpu_parity.py::test_four_step_long_lines);
// DFFT_NO_LONG_LINES=1 restores the "unsupported length" answer.
static int make_four_step(dfft_lines_plan p, int n, long long nlines)
{
    const int precision = p->prec;
    long long best1 = 0;
    int best_score = -1;
    for (long long d = 2; d * d <= (long long)n * 4 && d < n; d++) {
        if (n % d) continue;
        const SizeEntry *e1 = find_size_entry((int)d, precision), *e2 = find_size_entry((int)(n / d), precision);
        if (!e1 || !e2) continue;
        const long long q = n / d;
        const double ratio = d > q ? (double)d / q : (double)q / d;
        int score = (e1->gen ? 0 : 1000) + (e2->gen ? 0 : 1000) + (int)(500.0 / ratio);
        if (score > best_score) { best_score = score; best1 = d; }
    }
    if (!best1) return fail(DFFT_EUNSUPPORTED, "length %d cannot be split into two supported factors", n);
    if (!fits_int(nlines)) return fail(DFFT_EUNSUPPORTED, "%lld rows: at most 2^31 - 1 per plan", nlines);
    const int n1 = (int)best1, n2 = n / n1;
    p->temp_bytes = (size_t)nlines * n * (precision == DFFT_FLOAT ? 8 : 16);
    // pass A: columns of the [n1][n2] matrix of every line, transposed store + twiddle
    LinePass& a = p->run[0][0];
    a.e = find_size_entry(n1, precision);
    const int CA = a.e->x_C;
    a.G = (int)cdiv(n2, CA); a.W = n2; a.ntiles = nlines * a.G;
    a.ia = Affine{(long long)n, CA, 1, n2};
    a.oa = Affine{(long long)n, (long long)CA * n1, n1, 1};
    a.kind = PK_XF_TW; a.tw_n = n; a.src = LB_IN; a.dst = LB_TEMP;
    // pass B: columns of the [n2][n1] matrix in temp, natural-order result in the caller's buffer
    LinePass& b = p->run[0][1];
    b.e = find_size_entry(n2, precision);
    const int CB = b.e->s_C;
    b.G = (int)cdiv(n1, CB); b.W = n1; b.ntiles = nlines * b.G;
    b.ia = Affine{(long long)n, CB, 1, n1};
    b.oa = b.ia;
    b.kind = PK_Y; b.src = LB_TEMP; b.dst = LB_IN;
    return complex_lists(p, 2, true);
}

// 1-D lines in place (dfft_lines_plan_create): one pass, or, for a contiguous length beyond one shared-memory line and long_lines,
// the four-step pair
static int make_lines_1d(dfft_lines_plan p, int n, long long stride, long long nlines, long long inner, long long inner_dist, long long outer_dist,
                         bool long_lines)
{
    if (n < 1 || nlines < 0 || stride < 1 || bad_precision(p->prec)) return fail(DFFT_EINVAL, "bad arguments");
    if (long_lines && !find_size_entry(n, p->prec) && stride == 1 && inner_dist == n) {
        // the four-step passes address the lines as one dense block, as the contiguous pass does
        if (inner != nlines && outer_dist != inner * n) return fail(DFFT_EUNSUPPORTED, "contiguous lines must be densely packed");
        return make_four_step(p, n, nlines);
    }
    const int rc = make_line_pass(p->run[0][0], n, stride, nlines, inner, inner_dist, outer_dist, p->prec);
    return rc ? rc : complex_lists(p, 1, false);
}

// batch ny x nx matrices (nx fastest), in place: X along the batch*ny rows, Y over the nx columns of every matrix (stride nx);
// backward in reverse
static int make_lines_2d(dfft_lines_plan p, int nx, int ny, long long batch)
{
    if (nx < 1 || ny < 1 || batch < 0 || bad_precision(p->prec)) return fail(DFFT_EINVAL, "bad arguments");
    if (!fits_int(ny, batch)) return fail(DFFT_EUNSUPPORTED, "%d x %lld rows: at most 2^31 - 1 per plan", ny, batch);
    int rc = make_line_pass(p->run[0][0], nx, 1, (long long)ny * batch, (long long)ny * batch, nx, 0, p->prec);
    if (!rc) rc = make_line_pass(p->run[0][1], ny, nx, (long long)nx * batch, nx, 1, (long long)nx * ny, p->prec);
    return rc ? rc : complex_lists(p, 2, false);
}

static bool env_on(const char* name)
{
    const char* v = getenv(name);
    return v && atoi(v) != 0;
}

// batch nz x ny x nx volumes (nx fastest), in place: X along the batch*nz*ny rows, Y over the nx columns of every plane (stride
// nx), Z over the nx*ny columns of every volume (stride nx*ny); backward in reverse.  Where nx == ny and the entry has a plane
// kernel that is the default for its shape (plane_default; DFFT_FORCE_PLANE=1: wherever instantiated), X and Y are one launch
// of it over the batch*nz planes.  DFFT_NO_PLANE=1 keeps the separate passes.  Read at plan creation
static int make_lines_3d(dfft_lines_plan p, int nx, int ny, int nz, long long batch)
{
    const int precision = p->prec;
    if (nx < 1 || ny < 1 || nz < 1 || batch < 0 || bad_precision(precision)) return fail(DFFT_EINVAL, "bad arguments");
    if (!fits_int(ny, nz, batch)) return fail(DFFT_EUNSUPPORTED, "%d x %d x %lld rows: at most 2^31 - 1 per plan", ny, nz, batch);
    const long long planes = (long long)nz * batch, rows = planes * ny, plane = (long long)nx * ny;
    const SizeEntry* ex = find_size_entry(nx, precision);
    const bool use_plane = ex && nx == ny && ex->launch[PK_PLANE] && !env_on("DFFT_NO_PLANE") && (plane_default(nx, precision) || env_on("DFFT_FORCE_PLANE"));
    LinePass* f = p->run[0];
    int rc = 0, k = 0;
    if (use_plane) {
        LinePass& lp = f[k++];
        lp.e = ex; lp.kind = PK_PLANE; lp.ntiles = planes;
        lp.ia = lp.oa = Affine{plane, 0, nx, 1};
    } else {
        rc = make_line_pass(f[k++], nx, 1, rows, rows, nx, 0, precision);
        if (!rc) rc = make_line_pass(f[k++], ny, nx, nx * planes, nx, 1, plane, precision);
    }
    if (!rc) rc = make_line_pass(f[k++], nz, plane, plane * batch, plane, 1, plane * nz, precision);
    return rc ? rc : complex_lists(p, k, false);
}

// ---- real lines: R2C / C2R over densely packed lines (1-D) and the rows of row-major matrices (2-D) --------------------------
// The real pass is the kernel pair of the 3-D plan's Z pass (Pass<T>::z_real): two real lines per complex transform, lines
// paired in order, on the tuned kernels (fft_real.cuh) or, for a run-time-scheduled length, fft_generic_r2c / c2r_kernel.
static void make_real_pass(LinePass& lp, const SizeEntry* e, long long nlines, bool fwd, int src, int dst)
{
    const int C = e->z_C;
    const long long N = e->N, H = N / 2 + 1;
    lp.e = e;
    lp.kind = fwd ? PK_Z_R2C : PK_Z_C2R;
    lp.G = (int)cdiv(cdiv(nlines, 2), C); lp.ntiles = lp.G; lp.W = (int)nlines;
    const Affine rmap{0, 2LL * C * N, 2 * N, 1}, cmap{0, 2LL * C * H, 2 * H, 1};   // tile, pair and point strides of each side
    lp.ia = fwd ? rmap : cmap; lp.oa = fwd ? cmap : rmap;
    lp.ld_in = fwd ? N : H; lp.ld_out = fwd ? H : N;
    lp.src = src; lp.dst = dst;
}

// 1-D: `batch` lines of n points (ny, nz unused).  2-D: `batch` ny x n matrices, rows real <-> rows of n/2+1 complex points.
// 3-D: `batch` nz x ny x n volumes, likewise
static int make_real_lines(dfft_lines_plan p, int n, int ny, int nz, long long batch, int dims)
{
    const int precision = p->prec;
    if (batch < 0 || (dims >= 2 && ny < 1) || (dims == 3 && nz < 1) || bad_precision(precision)) return fail(DFFT_EINVAL, "bad arguments");
    const SizeEntry* e = n < 2 ? nullptr : find_size_entry(n, precision);
    if (!e) return fail(DFFT_EUNSUPPORTED, "real lines of %d points: the length must be 2..13-smooth and fit one shared-memory line", n);
    if (!e->launch[PK_Z_R2C] || !e->launch[PK_Z_C2R]) return fail(DFFT_EUNSUPPORTED, "the kernel entry of length %d has no real-data kernels", n);
    const long long my = dims >= 2 ? ny : 1, mz = dims == 3 ? nz : 1;
    if (!fits_int(my, mz, batch)) return fail(DFFT_EUNSUPPORTED, "%lld x %lld x %lld real lines: at most 2^31 - 1 per plan", my, mz, batch);
    const long long rows = my * mz * batch;
    const long long H = n / 2 + 1;
    p->form = LF_REAL;
    p->rcount = rows * n;
    p->ccount = rows * H;
    LinePass* f = p->run[0];
    LinePass* b = p->run[1];
    make_real_pass(f[0], e, rows, true, LB_IN, LB_OUT);
    if (dims == 1) {
        make_real_pass(b[0], e, rows, false, LB_IN, LB_OUT);
    } else {
        // along ny: the H columns of every half-spectrum matrix, matrices ny*H apart; along nz (3-D): the ny*H columns of every
        // volume, volumes nz*ny*H apart.  Forward in place in `out` after the real pass; backward the strided passes in reverse,
        // the first from `in` into the temporary, so that `in` is never written, the rest in place there
        const int ns = dims - 1;   // strided passes: f[1..ns] forward, b[0..ns-1] backward (the same passes in reverse)
        int rc = make_line_pass(f[1], ny, H, H * mz * batch, H, 1, H * ny, precision);
        if (!rc && dims == 3) rc = make_line_pass(f[2], nz, H * ny, H * ny * batch, H * ny, 1, H * ny * nz, precision);
        if (rc) return rc;
        for (int k = 1; k <= ns; k++) {
            f[k].src = f[k].dst = LB_OUT;
            b[ns - k] = f[k];
            b[ns - k].src = k == ns ? LB_IN : LB_TEMP; b[ns - k].dst = LB_TEMP;
        }
        make_real_pass(b[ns], e, rows, false, LB_TEMP, LB_OUT);
        p->temp_bytes = (size_t)p->ccount * (precision == DFFT_FLOAT ? 8 : 16);
    }
    p->nrun[0] = p->nrun[1] = dims;
    for (int k = 0; k < dims; k++) b[k].inv = true;
    return 0;
}

// ---- batched 2-D and 3-D spectral convolution on the lines engine: out = ifftn(fftn(in) * m) per image / volume ---------------
// The forward passes of the 2-D or 3-D lines plan (make_lines_2d / make_lines_3d / make_real_lines), the last one (Y in 2-D, Z in
// 3-D) replaced by PK_XCONV (forward, multiply, inverse in one column pass, as the slab convolve plan's X pass;
// fft_conv_shared_kernel when one multiplier serves every image / volume), then the forward passes before it again, inverse and
// in reverse order:
//   3-D C2C, plane kernel: XY_PLANE in -> out, XCONV, inverse XY_PLANE (6 volume sweeps + the multiplier)
//   3-D C2C, other shapes: X in -> out, Y, XCONV, inverse Y, inverse X (10 sweeps)
//   3-D R2C:               Z_R2C in -> temp, Y, XCONV, inverse Y, Z_C2R temp -> out
//   2-D C2C, plane conv:   XY_PLANE_CONV in -> out: the whole convolution of nx == ny images in one launch of launch[PK_PLANE_CONV]
//                          (plane_conv_default; DFFT_FORCE_PLANE=1: wherever instantiated; DFFT_NO_PLANE=1: never) (2 sweeps)
//   2-D C2C, other shapes: X in -> out, XCONV, inverse X (6 sweeps)
//   2-D R2C:               Z_R2C in -> temp, XCONV, Z_C2R temp -> out
// Everything after the first pass is in place in `out` (C2C) or the plan's temporary (R2C), so `in` is only read and in == out
// works.  The convolved length (ny in 2-D, nz in 3-D) needs the convolve kernel: a tuned default entry (launch[PK_XCONV], as
// dfft_plan_convolve_* asks of x)
static int make_lines_conv(dfft_lines_plan p, int dims, int nx, int ny, int nz, long long batch, bool real, unsigned flags)
{
    if (flags & ~DFFT_SCALE_BACKWARD) return fail(DFFT_EINVAL, "convolve lines plans take no flag but DFFT_SCALE_BACKWARD");
    const int rc = real ? make_real_lines(p, nx, ny, nz, batch, dims) : dims == 3 ? make_lines_3d(p, nx, ny, nz, batch) : make_lines_2d(p, nx, ny, batch);
    if (rc) return rc;
    const LinePass* f = p->run[0];   // forward passes in execution order, the convolved axis last
    const int nf = p->nrun[0];
    assert(nf >= 2 && nf <= 3);      // X + Y or the plane pass (2-D), then Z (3-D): the list below has 2 * nf - 1 <= 5 passes
    const LinePass& z = f[nf - 1];
    if (z.kind != PK_Y || z.e->gen || !z.e->launch[PK_XCONV])
        return fail(DFFT_EUNSUPPORTED, "the %c length %d has no convolution kernel (it needs a tuned length, dfft_length_kind == 2, of the default kernel table)",
                    dims == 3 ? 'z' : 'y', dims == 3 ? nz : ny);
    const int buf = real ? LB_TEMP : LB_OUT;
    LinePass c[5];
    int k = 0;
    for (int j = 0; j < nf; j++) {
        c[k] = f[j];
        c[k].src = j == 0 ? LB_IN : buf; c[k++].dst = buf;
    }
    c[nf - 1].kind = PK_XCONV;
    for (int j = nf - 2; j >= (real ? 1 : 0); j--) {
        c[k] = f[j];
        c[k].src = c[k].dst = buf; c[k++].inv = true;
    }
    const long long vol = (long long)nx * ny * (dims == 3 ? nz : 1);
    if (real) make_real_pass(c[k++], f[0].e, vol / nx * batch, false, LB_TEMP, LB_OUT);   // Z_C2R temp -> out
    if (dims == 2 && !real && nx == ny && f[0].e->launch[PK_PLANE_CONV] && !env_on("DFFT_NO_PLANE") && (plane_conv_default(nx, p->prec) || env_on("DFFT_FORCE_PLANE"))) {
        // the three passes become one, on the X pass's buffers and contiguous twiddle table (one Sched at these lengths)
        c[0].kind = PK_PLANE_CONV; c[0].ntiles = batch;
        c[0].ia = c[0].oa = Affine{(long long)nx * ny, 0, nx, 1};
        k = 1;
    }
    std::copy(c, c + k, p->run[0]);
    p->nrun[0] = k;
    p->nrun[1] = 0;
    p->form = LF_CONV;
    p->real = real;
    p->batch = batch;
    p->mvol = real ? vol / nx * (nx / 2 + 1) : vol;
    if (real) p->rcount = vol * batch;
    else p->ccount = vol * batch;
    p->scale = (flags & DFFT_SCALE_BACKWARD) ? 1.0 / (double)vol : 0.0;
    return 0;
}

// ---- batched 1-D spectral convolution on the lines engine: out = ifft(fft(in) * m) per line, or irfft(rfft(in) * m, n) -------
// `nlines` densely packed lines of n points, convolved in ONE pass in -> out: LINE_CONV (fft_line_conv_kernel, C lines per tile)
// or LINE_CONV_R2C (fft_line_conv_r2c_kernel, C line pairs per tile, as the real lines plan's R2C pass).  One sweep of the batch
// in, one out, and the multiplier.  n needs a tuned default entry (dfft_length_kind == 2); generic lengths and lines longer than
// one shared-memory line (the four-step plan) have no line-convolution kernel.  The plan needs no temporary
static int make_lines_conv_1d(dfft_lines_plan p, int n, long long nlines, bool real, unsigned flags)
{
    if (flags & ~DFFT_SCALE_BACKWARD) return fail(DFFT_EINVAL, "convolve lines plans take no flag but DFFT_SCALE_BACKWARD");
    if (n < 1 || nlines < 0 || bad_precision(p->prec)) return fail(DFFT_EINVAL, "bad arguments");
    if (real && n < 2) return fail(DFFT_EUNSUPPORTED, "real lines of %d points: a real convolution needs at least 2", n);
    const SizeEntry* e = find_size_entry(n, p->prec);
    if (!e || e->gen || !e->launch[real ? PK_LINE_CONV_R2C : PK_LINE_CONV])
        return fail(DFFT_EUNSUPPORTED, "length %d has no line-convolution kernel: it needs a tuned length (dfft_length_kind == 2) of the default "
                    "kernel table; generic lengths and lines longer than one shared-memory line are not convolved", n);
    if (!fits_int(nlines)) return fail(DFFT_EUNSUPPORTED, "%lld lines: at most 2^31 - 1 per plan", nlines);
    const int C = e->z_C;
    LinePass& lp = p->run[0][0];
    lp.e = e;
    lp.src = LB_IN; lp.dst = LB_OUT;
    lp.W = (int)nlines;
    if (real) {
        lp.kind = PK_LINE_CONV_R2C;
        lp.G = (int)cdiv(cdiv(nlines, 2), C);
        lp.ia = lp.oa = Affine{0, 2LL * C * n, 2LL * n, 1};   // tile, pair and point strides (reals)
        lp.ld_in = lp.ld_out = n;
    } else {
        lp.kind = PK_LINE_CONV;
        lp.G = (int)cdiv(nlines, C);
        lp.ia = lp.oa = Affine{0, (long long)C * n, n, 1};
    }
    lp.ntiles = lp.G;
    p->nrun[0] = 1;
    p->nrun[1] = 0;
    p->form = LF_CONV;
    p->real = real;
    p->batch = nlines;
    p->mvol = real ? n / 2 + 1 : n;
    if (real) p->rcount = nlines * n;
    else p->ccount = nlines * n;
    p->scale = (flags & DFFT_SCALE_BACKWARD) ? 1.0 / (double)n : 0.0;
    return 0;
}

static int lines_plan_common(dfft_lines_plan p, int precision)
{
    p->prec = precision;
    CU(cudaGetDevice(&p->device));
    CU(cudaDeviceGetAttribute(&p->sms, cudaDevAttrMultiProcessorCount, p->device));
    CU(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
    for (auto& e : p->ev) CU(cudaEventCreate(&e));
    return 0;
}

// the device twiddle table of lp's entry and schedule, uploaded in the plan's precision when a pass first asks for it
static int lines_lut(dfft_lines_plan p, LinePass& lp)
{
    const int kind = plain_kind(lp.kind);
    for (const auto& t : p->luts)
        if (t.e == lp.e && t.kind == kind) { lp.lut = t.d; return 0; }
    const cudaError_t err = p->prec == DFFT_DOUBLE ? upload_lut_kind<double>(&lp.lut, lp.e, kind) : upload_lut_kind<float>(&lp.lut, lp.e, kind);
    if (lp.lut) p->luts.push_back({lp.e, kind, lp.lut});
    if (err != cudaSuccess || !lp.lut) return fail(DFFT_ECUDA, "twiddle table upload failed");
    return 0;
}

extern "C" int dfft_lines_destroy(dfft_lines_plan p)
{
    if (!p) return 0;
    cudaSetDevice(p->device);
    if (p->stream) cudaStreamSynchronize(p->stream);
    for (const auto& t : p->luts) cudaFree(t.d);
    if (p->temp) cudaFree(p->temp);
    for (auto& e : p->ev) if (e) cudaEventDestroy(e);
    if (p->stream) cudaStreamDestroy(p->stream);
    cudaGetLastError();
    delete p;
    return 0;
}

// a plan laid out by `build` (which validates the arguments), with its twiddle tables and temporary; destroyed again on failure
template <class Build> static int lines_create(dfft_lines_plan* out, int precision, Build build)
{
    if (!out) return fail(DFFT_EINVAL, "null plan pointer");
    *out = nullptr;
    dfft_lines_plan p = new dfft_lines_plan_s;
    int rc = lines_plan_common(p, precision);
    if (!rc) rc = build(p);
    for (int d = 0; d < 2; d++)
        for (int k = 0; k < p->nrun[d] && !rc; k++) rc = lines_lut(p, p->run[d][k]);
    if (!rc && p->temp_bytes) {
        const cudaError_t err = cudaMalloc(&p->temp, p->temp_bytes);
        if (err != cudaSuccess) rc = fail(DFFT_ECUDA, "temporary allocation failed: %s", cudaGetErrorString(err));
    }
    if (rc) { dfft_lines_destroy(p); return rc; }
    *out = p;
    return 0;
}

extern "C" int dfft_lines_plan_create(int n, long long stride, long long nlines, long long inner, long long inner_dist, long long outer_dist,
                                      int precision, dfft_lines_plan* out)
{
    return lines_create(out, precision, [&](dfft_lines_plan p) {
        return make_lines_1d(p, n, stride, nlines, inner, inner_dist, outer_dist, !env_on("DFFT_NO_LONG_LINES"));
    });
}

/* batch of 2-D transforms, nx fastest: the reference's FFTdim = 2 application (Test_2D.cpp: size = {X, Y, Z}) */
extern "C" int dfft_lines_plan_create_2d(int nx, int ny, long long batch, int precision, dfft_lines_plan* out)
{
    return lines_create(out, precision, [&](dfft_lines_plan p) { return make_lines_2d(p, nx, ny, batch); });
}

extern "C" int dfft_lines_plan_create_3d(int nx, int ny, int nz, long long batch, int precision, dfft_lines_plan* out)
{
    return lines_create(out, precision, [&](dfft_lines_plan p) { return make_lines_3d(p, nx, ny, nz, batch); });
}

extern "C" int dfft_lines_plan_create_r2c(int n, long long nlines, int precision, dfft_lines_plan* plan)
{
    return lines_create(plan, precision, [&](dfft_lines_plan p) { return make_real_lines(p, n, 1, 1, nlines, 1); });
}

extern "C" int dfft_lines_plan_create_r2c_2d(int nx, int ny, long long batch, int precision, dfft_lines_plan* plan)
{
    return lines_create(plan, precision, [&](dfft_lines_plan p) { return make_real_lines(p, nx, ny, 1, batch, 2); });
}

extern "C" int dfft_lines_plan_create_r2c_3d(int nx, int ny, int nz, long long batch, int precision, dfft_lines_plan* plan)
{
    return lines_create(plan, precision, [&](dfft_lines_plan p) { return make_real_lines(p, nx, ny, nz, batch, 3); });
}

extern "C" int dfft_lines_plan_create_convolve_3d(int nx, int ny, int nz, long long batch, int precision, unsigned flags, dfft_lines_plan* plan)
{
    return lines_create(plan, precision, [&](dfft_lines_plan p) { return make_lines_conv(p, 3, nx, ny, nz, batch, false, flags); });
}

extern "C" int dfft_lines_plan_create_convolve_r2c_3d(int nx, int ny, int nz, long long batch, int precision, unsigned flags, dfft_lines_plan* plan)
{
    return lines_create(plan, precision, [&](dfft_lines_plan p) { return make_lines_conv(p, 3, nx, ny, nz, batch, true, flags); });
}

extern "C" int dfft_lines_plan_create_convolve_1d(int n, long long nlines, int precision, unsigned flags, dfft_lines_plan* plan)
{
    return lines_create(plan, precision, [&](dfft_lines_plan p) { return make_lines_conv_1d(p, n, nlines, false, flags); });
}

extern "C" int dfft_lines_plan_create_convolve_r2c_1d(int n, long long nlines, int precision, unsigned flags, dfft_lines_plan* plan)
{
    return lines_create(plan, precision, [&](dfft_lines_plan p) { return make_lines_conv_1d(p, n, nlines, true, flags); });
}

extern "C" int dfft_lines_plan_create_convolve_2d(int nx, int ny, long long batch, int precision, unsigned flags, dfft_lines_plan* plan)
{
    return lines_create(plan, precision, [&](dfft_lines_plan p) { return make_lines_conv(p, 2, nx, ny, 1, batch, false, flags); });
}

extern "C" int dfft_lines_plan_create_convolve_r2c_2d(int nx, int ny, long long batch, int precision, unsigned flags, dfft_lines_plan* plan)
{
    return lines_create(plan, precision, [&](dfft_lines_plan p) { return make_lines_conv(p, 2, nx, ny, 1, batch, true, flags); });
}

static inline void* line_buf(int which, const void* in, void* out, void* temp)
{
    return which == LB_TEMP ? temp : (which == LB_OUT ? out : const_cast<void*>(in));
}

// pass `lp` of a lines plan, at position `phase` of its list: launched on the plan's stream, or (ops) only recorded.  The one
// place that builds a lines pass's kernel arguments and its record; the launch path allocates nothing
template <typename T>
static cudaError_t line_pass(const dfft_lines_plan_s* p, const LinePass& lp, int phase, const void* in, void* out, const void* mult, bool shared,
                             std::vector<std::string>* ops = nullptr)
{
    const void* src = line_buf(lp.src, in, out, p->temp);
    void* dst = line_buf(lp.dst, in, out, p->temp);
    const bool conv = lp.kind == PK_XCONV || lp.kind == PK_PLANE_CONV || lp.kind == PK_LINE_CONV || lp.kind == PK_LINE_CONV_R2C;
    const bool realk = lp.kind == PK_Z_R2C || lp.kind == PK_Z_C2R || lp.kind == PK_LINE_CONV_R2C;
    ConvArgs<T> c{};
    TileArgs<T>& a = c.t;
    a.in = (const cx<T>*)src; a.out = (cx<T>*)dst; a.lut = (const cx<T>*)lp.lut;
    a.ia = lp.ia; a.oa = lp.oa; a.G = lp.G; a.W = lp.W; a.ntiles = lp.ntiles;
    a.inv = lp.inv; a.gen = lp.e->gen; a.tw_n = lp.tw_n;
    if (conv) {
        a.do_scale = p->scale != 0; a.scale = (T)p->scale;
        c.mult = (const cx<T>*)mult; c.mult_shared = shared ? 1 : 0;
    }
    if (ops) {
        char extra[192] = "";
        int len = 0;
        if (realk) len = snprintf(extra, sizeof(extra), ", \"nzh\": %d, \"pair\": [%lld, %lld]", lp.e->N / 2 + 1, lp.ld_in, lp.ld_out);
        if (conv) snprintf(extra + len, sizeof(extra) - len, ", \"mult\": %llu, \"shared\": %d", (unsigned long long)(size_t)mult, shared ? 1 : 0);
        const bool plane = lp.kind == PK_PLANE || lp.kind == PK_PLANE_CONV;
        record_op<T>(*ops, kPassNames[lp.kind], phase, lp.e->N, plane ? lp.e->N : kind_C(lp.e, plain_kind(lp.kind)), false, false, lp.kind == PK_XF_TW, a,
                     extra);
        return cudaSuccess;
    }
    // the kind's argument struct: the tile arguments (a), the column convolve's (c), or one of these
    PlaneConvArgs<T> pc{};      // PK_PLANE: pc.p
    RealLineConvArgs<T> rl{};   // PK_Z_R2C / PK_Z_C2R: rl.r
    LineConvArgs<T> lc{};
    const void* args = conv ? (const void*)&c : (const void*)&a;
    switch (lp.kind) {
    case PK_PLANE:
        pc.p = {a.in, a.out, a.lut, lp.ntiles, a.inv};
        args = &pc.p;
        break;
    case PK_PLANE_CONV:
        pc = {{a.in, a.out, a.lut, lp.ntiles, 0}, c.mult, shared ? 0 : (long long)lp.e->N * lp.e->N, a.scale, a.do_scale};
        args = &pc;
        break;
    case PK_Z_R2C: case PK_Z_C2R:
        rl.r = {a, (const T*)src, (T*)dst, lp.ld_in, lp.ld_out};
        args = &rl.r;
        break;
    case PK_LINE_CONV:
        lc = {a, c.mult, shared ? 0 : (long long)lp.e->N};
        args = &lc;
        break;
    case PK_LINE_CONV_R2C:
        rl = {{a, (const T*)src, (T*)dst, lp.ld_in, lp.ld_out}, c.mult, shared ? 0 : (long long)(lp.e->N / 2 + 1)};
        args = &rl;
        break;
    }
    return lp.e->launch[lp.kind](args, p->sms, p->stream);
}

// one execute: the passes of run[list] between the plan's two events
template <typename T> static int lines_run(dfft_lines_plan p, int list, const void* in, void* out, const void* mult = nullptr, bool shared = false)
{
    CU(cudaSetDevice(p->device));
    CU(cudaEventRecord(p->ev[0], p->stream));
    for (int k = 0; k < p->nrun[list]; k++) {
        const LinePass& lp = p->run[list][k];
        if (lp.ntiles <= 0) continue;
        const cudaError_t err = line_pass<T>(p, lp, k, in, out, mult, shared);
        if (err != cudaSuccess) return fail(DFFT_ECUDA, "line pass launch failed: %s", cudaGetErrorString(err));
    }
    CU(cudaEventRecord(p->ev[1], p->stream));
    return 0;
}

extern "C" int dfft_lines_execute(dfft_lines_plan p, void* data, int direction)
{
    if (!p || !data || (direction != DFFT_FORWARD && direction != DFFT_BACKWARD)) return fail(DFFT_EINVAL, "bad arguments");
    if (p->form == LF_CONV) return fail(DFFT_EINVAL, "a convolve lines plan runs with dfft_lines_execute_convolve");
    if (p->form == LF_REAL) return fail(DFFT_EINVAL, "a real lines plan runs with dfft_lines_execute_real");
    const int list = direction == DFFT_BACKWARD;
    return p->prec == DFFT_DOUBLE ? lines_run<double>(p, list, data, data) : lines_run<float>(p, list, data, data);
}

extern "C" int dfft_lines_execute_real(dfft_lines_plan p, const void* in, void* out, int direction)
{
    if (!p || !in || !out || (direction != DFFT_FORWARD && direction != DFFT_BACKWARD)) return fail(DFFT_EINVAL, "bad arguments");
    if (p->form == LF_CONV) return fail(DFFT_EINVAL, "a convolve lines plan runs with dfft_lines_execute_convolve");
    if (p->form != LF_REAL) return fail(DFFT_EINVAL, "a complex lines plan runs with dfft_lines_execute");
    const size_t rsz = p->prec == DFFT_FLOAT ? 4 : 8, csz = 2 * rsz;
    const bool fwd = direction == DFFT_FORWARD;
    const uintptr_t ri = (uintptr_t)(fwd ? in : out), ci = (uintptr_t)(fwd ? out : in);
    if (ri % rsz || ci % csz) return fail(DFFT_EINVAL, "a %s buffer is not aligned to its element size", ri % rsz ? "real" : "complex");
    const uintptr_t a = (uintptr_t)in, b = (uintptr_t)out;
    const uintptr_t a_end = a + (fwd ? p->rcount * rsz : p->ccount * csz), b_end = b + (fwd ? p->ccount * csz : p->rcount * rsz);
    if (a == b || (a < b_end && b < a_end)) return fail(DFFT_EINVAL, "`in` and `out` overlap (real lines are out of place)");
    const int list = fwd ? 0 : 1;
    return p->prec == DFFT_DOUBLE ? lines_run<double>(p, list, in, out) : lines_run<float>(p, list, in, out);
}

extern "C" int dfft_lines_execute_convolve(dfft_lines_plan p, const void* in, void* out, const void* mult, long long mult_count)
{
    if (!p || !in || !out || !mult) return fail(DFFT_EINVAL, "bad arguments");
    if (p->form != LF_CONV) return fail(DFFT_EINVAL, "dfft_lines_execute_convolve needs a plan from dfft_lines_plan_create_convolve_[r2c_]1d / _2d / _3d");
    if (mult_count != 1 && mult_count != p->batch) return fail(DFFT_EINVAL, "mult_count must be 1 or the plan's batch (%lld), not %lld", p->batch, mult_count);
    const bool real = p->real;
    const size_t rsz = p->prec == DFFT_FLOAT ? 4 : 8, csz = 2 * rsz, esz = real ? rsz : csz;
    const uintptr_t a = (uintptr_t)in, b = (uintptr_t)out, m = (uintptr_t)mult;
    if (a % esz || b % esz || m % csz) return fail(DFFT_EINVAL, "a buffer is not aligned to its element size");
    const uintptr_t io = (uintptr_t)((real ? p->rcount : p->ccount) * esz), mb = (uintptr_t)(mult_count * p->mvol * csz);
    if (a != b && a < b + io && b < a + io) return fail(DFFT_EINVAL, "`in` and `out` overlap without being the same buffer");
    if (m < b + io && b < m + mb) return fail(DFFT_EINVAL, "the multiplier overlaps `out`");
    const bool shared = mult_count == 1;
    return p->prec == DFFT_DOUBLE ? lines_run<double>(p, 0, in, out, mult, shared) : lines_run<float>(p, 0, in, out, mult, shared);
}

extern "C" int dfft_lines_synchronize(dfft_lines_plan p)
{
    if (!p) return fail(DFFT_EINVAL, "null plan");
    CU(cudaSetDevice(p->device));
    CU(cudaStreamSynchronize(p->stream));
    return 0;
}

extern "C" void* dfft_lines_stream(dfft_lines_plan p) { return p ? (void*)p->stream : nullptr; }

// the records of list `list` of the describe-only plan `build` lays out, in the hooks' JSON; buffers of device 0: `in`, `out`, the
// temporary 4, the multiplier 8
template <class Build> static long long lines_ops_json(int precision, Build build, int list, int in, int out, bool shared, char* buf, long long cap)
{
    dfft_lines_plan_s p;
    p.prec = precision;
    p.temp = fake_addr(0, 4);
    const int rc = build(&p);
    if (rc) return rc;
    std::vector<std::string> ops;
    for (int k = 0; k < p.nrun[list]; k++) line_pass<double>(&p, p.run[list][k], k, fake_addr(0, in), fake_addr(0, out), fake_addr(0, 8), shared, &ops);
    return ops_json(ops, buf, cap);
}

/* test hook (host only): the passes a lines plan would launch for `direction`, as JSON (same format as dfft_debug_plan_ops;
 * the caller's data is buffer 1 of device 0, the plan's temporary buffer 4); two_d != 0: 2-D plan (n = nx, stride = ny,
 * nlines = batch).  Long lines always use the four-step plan here.  Returns the bytes needed, < 0 on error. */
extern "C" long long dfft_debug_lines_ops(int n, long long stride, long long nlines, long long inner, long long inner_dist, long long outer_dist,
                                          int precision, int direction, int two_d, char* buf, long long cap)
{
    auto build = [&](dfft_lines_plan p) {
        return two_d ? make_lines_2d(p, n, (int)stride, nlines) : make_lines_1d(p, n, stride, nlines, inner, inner_dist, outer_dist, true);
    };
    return lines_ops_json(precision, build, direction == DFFT_BACKWARD, 1, 1, false, buf, cap);
}

/* test hook (host only): the passes of a real lines plan for `direction`, JSON as dfft_debug_lines_ops; in = buffer 5, out = 2,
 * temporary = 4 of device 0.  Real passes carry "nzh" and "pair" as the 3-D plan's Z_R2C / Z_C2R records */
extern "C" long long dfft_debug_real_lines_ops(int n, int ny, long long batch, int precision, int direction, int two_d, char* buf, long long cap)
{
    if (direction != DFFT_FORWARD && direction != DFFT_BACKWARD) return fail(DFFT_EINVAL, "bad direction");
    auto build = [&](dfft_lines_plan p) { return make_real_lines(p, n, ny, 1, batch, two_d ? 2 : 1); };
    return lines_ops_json(precision, build, direction == DFFT_BACKWARD, 5, 2, false, buf, cap);
}

/* test hook (host only): the passes of a 3-D lines plan for `direction`, JSON as dfft_debug_lines_ops (complex: the caller's data
 * is buffer 1) or dfft_debug_real_lines_ops (real != 0: in = buffer 5, out = 2, temporary = 4).  The plane kernel's record is
 * "XY_PLANE" with ntiles = planes and ia = oa = [plane, 0, row, point] strides */
extern "C" long long dfft_debug_lines_3d_ops(int nx, int ny, int nz, long long batch, int precision, int direction, int real, char* buf, long long cap)
{
    if (direction != DFFT_FORWARD && direction != DFFT_BACKWARD) return fail(DFFT_EINVAL, "bad direction");
    auto build = [&](dfft_lines_plan p) { return real ? make_real_lines(p, nx, ny, nz, batch, 3) : make_lines_3d(p, nx, ny, nz, batch); };
    return lines_ops_json(precision, build, direction == DFFT_BACKWARD, real ? 5 : 1, real ? 2 : 1, false, buf, cap);
}

/* test hook (host only): the passes of a convolve lines plan, JSON as dfft_debug_lines_3d_ops; in = buffer 5, out = 2,
 * temporary = 4, multiplier = 8 of device 0.  XCONV carries "mult" and "shared" (1: mult_count == 1) */
extern "C" long long dfft_debug_lines_conv_3d_ops(int nx, int ny, int nz, long long batch, int precision, int real, unsigned flags,
                                                  long long mult_count, char* buf, long long cap)
{
    auto build = [&](dfft_lines_plan p) {
        const int rc = make_lines_conv(p, 3, nx, ny, nz, batch, real != 0, flags);
        return rc || mult_count == 1 || mult_count == batch ? rc : fail(DFFT_EINVAL, "mult_count must be 1 or the plan's batch");
    };
    return lines_ops_json(precision, build, 0, 5, 2, mult_count == 1, buf, cap);
}

/* test hook (host only): the passes of a 2-D convolve lines plan, JSON as dfft_debug_lines_conv_3d_ops.  The plane-convolve
 * kernel's record is "XY_PLANE_CONV" with ntiles = images, ia = oa = [image, 0, row, point] strides, "mult" and "shared" */
extern "C" long long dfft_debug_lines_conv_2d_ops(int nx, int ny, long long batch, int precision, int real, unsigned flags,
                                                  long long mult_count, char* buf, long long cap)
{
    auto build = [&](dfft_lines_plan p) {
        const int rc = make_lines_conv(p, 2, nx, ny, 1, batch, real != 0, flags);
        return rc || mult_count == 1 || mult_count == batch ? rc : fail(DFFT_EINVAL, "mult_count must be 1 or the plan's batch");
    };
    return lines_ops_json(precision, build, 0, 5, 2, mult_count == 1, buf, cap);
}

/* test hook (host only): the pass of a 1-D convolve lines plan, JSON as dfft_debug_lines_conv_3d_ops (in = buffer 5, out = 2,
 * multiplier = 8 of device 0).  The record is "LINE_CONV" (real != 0: "LINE_CONV_R2C", which also carries "nzh" and "pair") with
 * C = lines (line pairs) per tile, G = ntiles tiles, W = lines, "mult" and "shared" */
extern "C" long long dfft_debug_lines_conv_1d_ops(int n, long long nlines, int precision, int real, unsigned flags, long long mult_count,
                                                  char* buf, long long cap)
{
    auto build = [&](dfft_lines_plan p) {
        const int rc = make_lines_conv_1d(p, n, nlines, real != 0, flags);
        return rc || mult_count == 1 || mult_count == nlines ? rc : fail(DFFT_EINVAL, "mult_count must be 1 or the plan's line count");
    };
    return lines_ops_json(precision, build, 0, 5, 2, mult_count == 1, buf, cap);
}

extern "C" int dfft_fft_lines(void* data, int n, long long stride, long long nlines, long long inner, long long inner_dist,
                              long long outer_dist, int direction, int precision)
{
    if (!data || n < 1 || nlines < 0 || stride < 1) return fail(DFFT_EINVAL, "bad arguments");
    if (direction != DFFT_FORWARD && direction != DFFT_BACKWARD) return fail(DFFT_EINVAL, "direction must be +1 or -1");
    if (nlines == 0) return 0;
    dfft_lines_plan p = nullptr;
    int rc = dfft_lines_plan_create(n, stride, nlines, inner, inner_dist, outer_dist, precision, &p);
    if (rc) return rc;
    rc = dfft_lines_execute(p, data, direction);
    if (!rc) rc = dfft_lines_synchronize(p);
    dfft_lines_destroy(p);
    return rc;
}
