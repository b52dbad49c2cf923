// fake_cudart.cpp -- TEST INFRASTRUCTURE ONLY.  A stand-in for the CUDA runtime entry points libdfft.so
// uses: device memory is host memory, copies are memcpy, kernel launches are counted no-ops, events and
// streams are dummies.  tests/test_control_flow_fakecuda.py links the library's own objects against this
// file (nvcc -cudart none) so that a NON-dry plan can be driven create -> execute -> timings -> destroy
// on a box without a GPU: host-side hangs, recursion and bootstrap deadlocks show up in seconds.
// Nothing on the product path links or loads this file.
#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

extern "C" {

typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
struct dim3_ { unsigned x, y, z; };
struct cudaIpcMemHandle_st { char reserved[64]; };

static std::atomic<long long> g_launches{0}, g_events{0}, g_mallocs{0}, g_frees{0};
static thread_local int t_device = 0;
static thread_local dim3_ t_grid, t_block;
static thread_local size_t t_smem;
static thread_local cudaStream_t t_stream;

long long fakecuda_launches(void) { return g_launches.load(); }
long long fakecuda_event_records(void) { return g_events.load(); }
long long fakecuda_live_allocations(void) { return g_mallocs.load() - g_frees.load(); }

// --- registration hooks emitted by nvcc for every translation unit with kernels
void** __cudaRegisterFatBinary(void*) { static void* h; return &h; }
void __cudaRegisterFatBinaryEnd(void**) {}
void __cudaUnregisterFatBinary(void**) {}
void __cudaRegisterFunction(void**, const char*, char*, const char*, int, void*, void*, void*, void*, int*) {}
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
cudaError_t cudaLaunchKernel(const void*, dim3_ grid, dim3_ block, void**, size_t, cudaStream_t)
{
    if (grid.x == 0 || block.x == 0 || block.x * block.y * block.z > 1024) return 9;   // cudaErrorInvalidConfiguration
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
cudaError_t cudaGetLastError(void) { return 0; }
const char* cudaGetErrorString(cudaError_t e) { return e ? "fake CUDA error" : "no error"; }
cudaError_t cudaFuncSetAttribute(const void*, int, int) { return 0; }
cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(int* n, const void*, int, size_t, unsigned) { *n = 2; return 0; }

// --- memory: plain host memory (sizes are test-sized)
cudaError_t cudaMalloc(void** p, size_t n) { *p = calloc(1, n ? n : 1); g_mallocs++; return *p ? 0 : 2; }
cudaError_t cudaMallocHost(void** p, size_t n) { *p = calloc(1, n ? n : 1); g_mallocs++; return *p ? 0 : 2; }
cudaError_t cudaFree(void* p) { if (p) g_frees++; free(p); return 0; }
cudaError_t cudaFreeHost(void* p) { if (p) g_frees++; free(p); return 0; }
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, int) { if (d != s) memmove(d, s, n); return 0; }
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t) { if (d != s) memmove(d, s, n); return 0; }
cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return 0; }
cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { memset(d, v, n); return 0; }
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_st* h, void* p) { memset(h, 0, sizeof(*h)); memcpy(h->reserved, &p, sizeof(p)); return 0; }
cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_st h, unsigned) { memcpy(p, h.reserved, sizeof(*p)); return 0; }
cudaError_t cudaIpcCloseMemHandle(void*) { return 0; }

// --- streams and events
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = malloc(8); return 0; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return 0; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return 0; }
cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = malloc(8); return 0; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = malloc(8); return 0; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return 0; }
cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { g_events++; return 0; }
cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.25f; return 0; }
cudaError_t cudaGetDriverEntryPoint(const char*, void** fn, unsigned long long, void*) { *fn = nullptr; return 0; }
cudaError_t cudaGetDriverEntryPointByVersion(const char*, void** fn, unsigned, unsigned long long, void*) { *fn = nullptr; return 0; }
}
