// fake_cudart.cpp -- TEST INFRASTRUCTURE ONLY.  A stand-in for the CUDA runtime entry points libdfft.so
// uses: device memory is host memory, copies are memcpy, kernel launches are counted no-ops, events and
// streams are dummies; launches, event records, stream waits and async copies are logged per host thread
// (fakecuda_trace).  tests/test_control_flow_fakecuda.py links the library's own objects against this
// file (nvcc -cudart none) so that a NON-dry plan can be driven create -> execute -> timings -> destroy
// on a box without a GPU: host-side hangs, recursion and bootstrap deadlocks show up in seconds.
// Nothing on the product path links or loads this file.
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

extern "C" {

typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
struct dim3_ { unsigned x, y, z; };
struct cudaIpcMemHandle_st { char reserved[64]; };

static std::atomic<long long> g_launches{0}, g_events{0}, g_mallocs{0}, g_frees{0};
static thread_local dim3_ t_grid, t_block;
static thread_local size_t t_smem;
static thread_local cudaStream_t t_stream;

long long fakecuda_launches(void) { return g_launches.load(); }
long long fakecuda_event_records(void) { return g_events.load(); }
long long fakecuda_live_allocations(void) { return g_mallocs.load() - g_frees.load(); }

// --- issue-order trace of the calling host thread: kernel launches (device name, grid, block, dynamic shared memory, stream),
// event records, stream waits, async copies and sets.  Streams and events are numbered per thread in creation order since the
// last fakecuda_trace_reset (0 = the legacy default stream), so two runs of the same schedule give the same text.
// function-local statics: __cudaRegisterFunction runs from the library's static initialisers, possibly before this file's
static std::mutex& names_mu() { static std::mutex m; return m; }
static std::map<const void*, std::string>& kernel_names() { static std::map<const void*, std::string> m; return m; }   // host stub -> device name
static std::map<const void*, int>& ordinals() { static std::map<const void*, int> m; return m; }   // stream / event -> ordinal in its creating thread
static thread_local std::string t_trace;
static thread_local int t_next_stream = 1, t_next_event = 1;

static void number(const void* h, int& next)
{
    std::lock_guard<std::mutex> g(names_mu());
    ordinals()[h] = next++;
}
static int ordinal(const void* h)
{
    if (!h) return 0;
    std::lock_guard<std::mutex> g(names_mu());
    auto it = ordinals().find(h);
    return it == ordinals().end() ? -1 : it->second;
}
static void trace(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
static void trace(const char* fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    t_trace += buf;
    t_trace += '\n';
}
// the calling thread's trace, one line per call; returns the bytes needed (with the terminating zero)
long long fakecuda_trace(char* buf, long long cap)
{
    const long long n = (long long)t_trace.size() + 1;
    if (buf && cap >= n) memcpy(buf, t_trace.c_str(), (size_t)n);
    return n;
}
void fakecuda_trace_reset(void)
{
    t_trace.clear();
    t_next_stream = t_next_event = 1;
}

// --- registration hooks emitted by nvcc for every translation unit with kernels
void** __cudaRegisterFatBinary(void*) { static void* h; return &h; }
void __cudaRegisterFatBinaryEnd(void**) {}
void __cudaUnregisterFatBinary(void**) {}
void __cudaRegisterFunction(void**, const char* stub, char*, const char* name, int, void*, void*, void*, void*, int*)
{
    std::lock_guard<std::mutex> g(names_mu());
    kernel_names()[stub] = name;
}
unsigned __cudaPushCallConfiguration(dim3_ grid, dim3_ block, size_t smem, cudaStream_t st)
{
    t_grid = grid; t_block = block; t_smem = smem; t_stream = st;
    return 0;
}
cudaError_t __cudaPopCallConfiguration(dim3_* grid, dim3_* block, size_t* smem, void* st)
{
    *grid = t_grid; *block = t_block; *smem = t_smem; *(cudaStream_t*)st = t_stream;
    return 0;
}
// The fold fields of a TileArgs (fft_passes.cuh), which leads the first one to three kernel parameters: completion signal and
// start gate carried by a pass kernel.  From `ci` on the layout is the same for both precisions.
struct ChunkTabMirror { void* cptr[32]; long long SAq[32]; int ediv, nchunks; };
struct TileArgsMirror {
    const void *in, *out, *lut;
    long long ia[4], oa[4], ntiles;
    int G, W;
    double scale;
    int inv, do_scale;
    ChunkTabMirror ci, co;
    const void* gen;
    long long tw_n;
    unsigned long long* sig[32];
    unsigned long long sig_val;
    unsigned int* done_ctr;
    int sig_n;
    const unsigned long long* wait_flags;
    unsigned long long wait_val;
    int wait_n;
    int max_ctas_per_sm;
};
static long long alloc_offset(const void* ptr);
static int tile_args_params(const std::string& name)
{
    if (name.find("fft_fused3_kernel") != std::string::npos) return 3;
    if (name.find("fft_fused2_kernel") != std::string::npos || name.find("fft_fused_yx_kernel") != std::string::npos) return 2;
    for (const char* k : {"fft_tile_kernel", "fft_generic_kernel", "fft_conv_kernel", "fft_z_r2c_kernel", "fft_z_c2r_kernel",
                          "fft_generic_r2c_kernel", "fft_generic_c2r_kernel"})
        if (name.find(k) != std::string::npos) return 1;
    return 0;
}

// --- launch set-up per (device, kernel stub), the device being the calling thread's current one: the dynamic shared-memory limit
// raised with cudaFuncSetAttribute(cudaFuncAttributeMaxDynamicSharedMemorySize), and how often the limit was raised, the
// occupancy queried and the kernel launched.  As on the real runtime, a launch asking for more than 48 KiB of dynamic shared
// memory fails unless this device's limit for the kernel covers it; a <<<>>> launch reports that through cudaGetLastError.
// Not traced: the golden traces stay as they are
struct LaunchSetup { long long smem_limit, attr_calls, occ_queries, launches; };
static std::mutex& setup_mu() { static std::mutex m; return m; }
static std::map<std::pair<int, const void*>, LaunchSetup>& setups() { static std::map<std::pair<int, const void*>, LaunchSetup> m; return m; }
static thread_local int t_device = 0;
static thread_local cudaError_t t_last_error = 0;

// one line per (device, kernel): "device attr_calls occ_queries launches name"; returns the bytes needed (with the terminating zero)
long long fakecuda_launch_setup(char* buf, long long cap)
{
    std::string o;
    {
        std::lock_guard<std::mutex> g(setup_mu());
        for (const auto& kv : setups()) {
            char line[64];
            snprintf(line, sizeof(line), "%d %lld %lld %lld ", kv.first.first, kv.second.attr_calls, kv.second.occ_queries, kv.second.launches);
            std::lock_guard<std::mutex> n(names_mu());
            auto it = kernel_names().find(kv.first.second);
            o += line + (it == kernel_names().end() ? std::string("?") : it->second) + "\n";
        }
    }
    const long long n = (long long)o.size() + 1;
    if (buf && cap >= n) memcpy(buf, o.c_str(), (size_t)n);
    return n;
}

cudaError_t cudaLaunchKernel(const void* stub, dim3_ grid, dim3_ block, void** args, size_t smem, cudaStream_t st)
{
    if (grid.x == 0 || block.x == 0 || block.x * block.y * block.z > 1024) return 9;   // cudaErrorInvalidConfiguration
    {
        std::lock_guard<std::mutex> g(setup_mu());
        LaunchSetup& s = setups()[{t_device, stub}];
        if (smem > 48 * 1024 && (long long)smem > s.smem_limit) return t_last_error = 1;   // cudaErrorInvalidValue
        s.launches++;
    }
    std::string name = "?";
    {
        std::lock_guard<std::mutex> g(names_mu());
        auto it = kernel_names().find(stub);
        if (it != kernel_names().end()) name = it->second;
    }
    trace("launch %s grid %u,%u,%u block %u,%u,%u smem %zu stream %d", name.c_str(), grid.x, grid.y, grid.z, block.x, block.y, block.z, smem,
          ordinal(st));
    // flag words are given as byte offsets into their allocation (SyncBlock: ready[32], arrive[32], part_arrive[..][32])
    if (name.find("signal_flags_kernel") != std::string::npos) {
        const unsigned long long* const* dst = (const unsigned long long* const*)args[0];
        trace("  signal n %d value %llu word +%lld", *(const int*)args[1], *(const unsigned long long*)args[2], alloc_offset(dst[0]));
    } else if (name.find("wait_flags_kernel") != std::string::npos) {
        trace("  wait n %d value %llu words +%lld", *(const int*)args[1], *(const unsigned long long*)args[2],
              alloc_offset(*(const void* const*)args[0]));
    }
    for (int i = 0, n = tile_args_params(name); i < n; i++) {
        const TileArgsMirror* a = (const TileArgsMirror*)args[i];
        if (a->sig_n > 0)
            trace("  param %d signals n %d value %llu word +%lld done_ctr +%lld", i, a->sig_n, a->sig_val, alloc_offset(a->sig[0]),
                  alloc_offset(a->done_ctr));
        if (a->wait_n > 0) trace("  param %d waits n %d value %llu words +%lld", i, a->wait_n, a->wait_val, alloc_offset(a->wait_flags));
    }
    g_launches++;
    return 0;
}

// --- devices
cudaError_t cudaGetDeviceCount(int* n) { const char* e = getenv("FAKECUDA_DEVICES"); *n = e ? atoi(e) : 8; return 0; }
cudaError_t cudaGetDevice(int* d) { *d = t_device; return 0; }
cudaError_t cudaSetDevice(int d) { t_device = d; return 0; }
cudaError_t cudaDeviceGetAttribute(int* v, int, int) { *v = 132; return 0; }
cudaError_t cudaDeviceSynchronize(void) { return 0; }
cudaError_t cudaDeviceCanAccessPeer(int* can, int, int) { *can = 1; return 0; }
cudaError_t cudaDeviceEnablePeerAccess(int, unsigned) { return 0; }
cudaError_t cudaGetLastError(void) { const cudaError_t e = t_last_error; t_last_error = 0; return e; }
const char* cudaGetErrorString(cudaError_t e) { return e ? "fake CUDA error" : "no error"; }
cudaError_t cudaFuncSetAttribute(const void* stub, int attr, int value)
{
    if (attr == 8) {   // cudaFuncAttributeMaxDynamicSharedMemorySize
        std::lock_guard<std::mutex> g(setup_mu());
        LaunchSetup& s = setups()[{t_device, stub}];
        s.smem_limit = value;
        s.attr_calls++;
    }
    return 0;
}
cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(int* n, const void* stub, int, size_t, unsigned)
{
    std::lock_guard<std::mutex> g(setup_mu());
    setups()[{t_device, stub}].occ_queries++;
    *n = 2;
    return 0;
}

// --- memory: plain host memory (sizes are test-sized)
static std::mutex& allocs_mu() { static std::mutex m; return m; }
static std::map<const char*, size_t>& allocs() { static std::map<const char*, size_t> m; return m; }   // device allocations: base -> bytes
static long long alloc_offset(const void* ptr)
{
    std::lock_guard<std::mutex> g(allocs_mu());
    auto it = allocs().upper_bound((const char*)ptr);
    if (it == allocs().begin()) return -1;
    --it;
    const long long off = (const char*)ptr - it->first;
    return off < (long long)it->second ? off : -1;
}
cudaError_t cudaMalloc(void** p, size_t n)
{
    *p = calloc(1, n ? n : 1);
    g_mallocs++;
    if (!*p) return 2;
    std::lock_guard<std::mutex> g(allocs_mu());
    allocs()[(const char*)*p] = n ? n : 1;
    return 0;
}
cudaError_t cudaMallocHost(void** p, size_t n) { *p = calloc(1, n ? n : 1); g_mallocs++; return *p ? 0 : 2; }
cudaError_t cudaFree(void* p)
{
    if (p) {
        g_frees++;
        std::lock_guard<std::mutex> g(allocs_mu());
        allocs().erase((const char*)p);
    }
    free(p);
    return 0;
}
cudaError_t cudaFreeHost(void* p) { if (p) g_frees++; free(p); return 0; }
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, int) { if (d != s) memmove(d, s, n); return 0; }
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int kind, cudaStream_t st)
{
    trace("memcpy_async %zu kind %d stream %d", n, kind, ordinal(st));
    if (d != s) memmove(d, s, n);
    return 0;
}
cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return 0; }
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t st)
{
    trace("memset_async %zu value %d stream %d", n, v, ordinal(st));
    memset(d, v, n);
    return 0;
}
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_st* h, void* p) { memset(h, 0, sizeof(*h)); memcpy(h->reserved, &p, sizeof(p)); return 0; }
cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_st h, unsigned) { memcpy(p, h.reserved, sizeof(*p)); return 0; }
cudaError_t cudaIpcCloseMemHandle(void*) { return 0; }

// --- streams and events
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = malloc(8); number(*s, t_next_stream); return 0; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return 0; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
cudaError_t cudaStreamWaitEvent(cudaStream_t st, cudaEvent_t e, unsigned)
{
    trace("wait stream %d event %d", ordinal(st), ordinal(e));
    return 0;
}
cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = malloc(8); number(*e, t_next_event); return 0; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = malloc(8); number(*e, t_next_event); return 0; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return 0; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t st)
{
    trace("record event %d stream %d", ordinal(e), ordinal(st));
    g_events++;
    return 0;
}
cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.25f; return 0; }
// --- tensor maps (FAKECUDA_TMA=1): a stand-in for cuTensorMapEncodeTiled that enforces the driver's documented constraints on
// the maps the library encodes (rank 3 here, 16-byte-aligned base, strides multiples of 16 bytes, box dims 1..256 and within
// their dims, inner box row a multiple of 16 bytes) and logs each one.  Without FAKECUDA_TMA there is no driver entry point,
// as before, and the library runs no TMA kernel.
struct TmaMapLog { long long ok, dtype, base_mod16, dims[3], strides[2], box[3]; };
static std::mutex g_tma_mu;
static std::vector<TmaMapLog> g_tma_log;

static int fake_encode_tiled(void* map, int dtype, unsigned rank, void* base, const unsigned long long* dims, const unsigned long long* strides,
                             const unsigned* box, const unsigned* estr, int, int, int, int)
{
    TmaMapLog l{};
    l.dtype = dtype;
    l.base_mod16 = (long long)((uintptr_t)base & 15);
    const long long esize = dtype == 8 ? 8 : dtype == 7 ? 4 : 0;   // CU_TENSOR_MAP_DATA_TYPE_FLOAT64 / FLOAT32
    bool ok = rank == 3 && esize != 0 && l.base_mod16 == 0 && map != nullptr;
    for (unsigned i = 0; i < 3 && i < rank; i++) {
        l.dims[i] = (long long)dims[i];
        l.box[i] = box[i];
        ok = ok && box[i] >= 1 && box[i] <= 256 && box[i] <= dims[i] && estr[i] == 1;
        if (i < 2) { l.strides[i] = (long long)strides[i]; ok = ok && strides[i] % 16 == 0; }
    }
    ok = ok && (box[0] * esize) % 16 == 0;
    l.ok = ok;
    if (map) memset(map, 0, 128);
    std::lock_guard<std::mutex> g(g_tma_mu);
    g_tma_log.push_back(l);
    return ok ? 0 : 1;   // CUDA_ERROR_INVALID_VALUE
}
// maps encoded since the last reset, 11 values each (ok, dtype, base mod 16, dims[3], strides[2], box[3])
long long fakecuda_tma_maps(long long* out, long long cap)
{
    std::lock_guard<std::mutex> g(g_tma_mu);
    const long long n = (long long)g_tma_log.size();
    for (long long i = 0; i < n && (i + 1) * 11 <= cap; i++) {
        const TmaMapLog& l = g_tma_log[i];
        const long long v[11] = {l.ok, l.dtype, l.base_mod16, l.dims[0], l.dims[1], l.dims[2], l.strides[0], l.strides[1], l.box[0], l.box[1], l.box[2]};
        memcpy(out + i * 11, v, sizeof(v));
    }
    return n;
}
void fakecuda_tma_reset(void) { std::lock_guard<std::mutex> g(g_tma_mu); g_tma_log.clear(); }

cudaError_t cudaGetDriverEntryPoint(const char* name, void** fn, unsigned long long, int* query)
{
    const char* e = getenv("FAKECUDA_TMA");
    if (e && atoi(e) != 0 && name && !strcmp(name, "cuTensorMapEncodeTiled")) {
        *fn = (void*)fake_encode_tiled;
        if (query) *query = 0;   // cudaDriverEntryPointSuccess
        return 0;
    }
    *fn = nullptr;
    return 0;
}
cudaError_t cudaGetDriverEntryPointByVersion(const char*, void** fn, unsigned, unsigned long long, void*) { *fn = nullptr; return 0; }
}
