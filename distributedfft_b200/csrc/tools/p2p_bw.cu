// p2p_bw.cu -- developer micro-benchmark (not part of the product path): how fast can one GPU WRITE into a peer's
// memory over NVLink, as a function of the store mechanism and of the contiguous run per row?  Answers which store
// shape the exchange-fused Y role should use.   usage: p2p_bw [MiB]   (needs 2 GPUs with peer access)
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// (1) fully contiguous: every warp instruction writes 512 contiguous bytes
__global__ void st_contig(double2* dst, long long n)
{
    const double2 v = make_double2(1.0, 2.0);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) __stcg(dst + i, v);
}
// (2) row segments: the buffer is rows of ROWLEN complex; a tile = SEG columns x 512 rows; a warp instruction covers
// 32 / SEG rows x SEG columns (SEG * 16 bytes contiguous per row) -- the Y role's store shape
template <int SEG> __global__ void st_rows(double2* dst, int rowlen, long long nrows)
{
    const double2 v = make_double2(1.0, 2.0);
    const int c = threadIdx.x % SEG, t = threadIdx.x / SEG, TT = blockDim.x / SEG;
    const int tiles_per_band = rowlen / SEG;
    const long long bands = nrows / 512, ntiles = bands * tiles_per_band;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long band = tile / tiles_per_band;
        const int b = (int)(tile % tiles_per_band);
        double2* p = dst + (band * 512) * rowlen + b * SEG + c;
        for (int r = t; r < 512; r += TT) __stcg(p + (long long)r * rowlen, v);
    }
}
// (3) TMA bulk stores of CHUNK contiguous bytes from shared memory
template <int CHUNK> __global__ void st_bulk(char* dst, long long bytes)
{
    extern __shared__ __align__(128) char sm[];
    for (int i = threadIdx.x; i < CHUNK / 16; i += blockDim.x) reinterpret_cast<double2*>(sm)[i] = make_double2(1.0, 2.0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0) {
        const long long nch = bytes / CHUNK;
        int k = 0;
        for (long long i = blockIdx.x; i < nch; i += gridDim.x) {
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst + i * CHUNK), "r"(smem_u32(sm)), "r"(CHUNK) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            if (++k % 8 == 0) asm volatile("cp.async.bulk.wait_group.read 4;" ::: "memory");
        }
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}
// (4) TMA tensor stores: box = SEG complex columns x 256 rows of a row-major matrix (row pitch = rowlen complex)
__global__ void st_tensor(const __grid_constant__ CUtensorMap map, int seg, int rowlen, long long nrows)
{
    extern __shared__ __align__(128) char sm[];
    const int box_bytes = seg * 16 * 256;
    for (int i = threadIdx.x; i < box_bytes / 16; i += blockDim.x) reinterpret_cast<double2*>(sm)[i] = make_double2(1.0, 2.0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0) {
        const int per_band = rowlen / seg;
        const long long bands = nrows / 256, n = bands * per_band;
        int k = 0;
        for (long long i = blockIdx.x; i < n; i += gridDim.x) {
            const int c0 = (int)(i % per_band) * seg * 2, c1 = (int)(i / per_band) * 256;
            asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"(&map), "r"(c0), "r"(c1), "r"(smem_u32(sm)) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            if (++k % 8 == 0) asm volatile("cp.async.bulk.wait_group.read 4;" ::: "memory");
        }
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

template <class F> static void timeit(const char* name, double bytes, F&& launch)
{
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    launch(); launch();
    CK(cudaDeviceSynchronize());
    cudaEventRecord(e0);
    for (int i = 0; i < 5; i++) launch();
    cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
    float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 5;
    printf("%-64s %8.3f ms  %7.1f GB/s\n", name, ms, bytes / ms * 1e-6);
    fflush(stdout);
}

int main(int argc, char** argv)
{
    const long long mib = argc > 1 ? atoll(argv[1]) : 512;
    int ndev = 0; CK(cudaGetDeviceCount(&ndev));
    if (ndev < 2) { printf("needs 2 GPUs\n"); return 0; }
    const long long bytes = mib << 20, n = bytes / 16;
    const int rowlen = 512; const long long nrows = n / rowlen;
    double2 *local, *peer;
    CK(cudaSetDevice(1)); CK(cudaMalloc(&peer, bytes));
    CK(cudaSetDevice(0)); CK(cudaMalloc(&local, bytes));
    int can = 0; CK(cudaDeviceCanAccessPeer(&can, 0, 1));
    if (!can) { printf("no peer access\n"); return 0; }
    CK(cudaDeviceEnablePeerAccess(1, 0));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    printf("%s x2, %lld MiB per test, %d SMs\n", prop.name, mib, sms);
    EncodeTiledFn enc = nullptr; cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&enc, cudaEnableDefault, &q));
    for (int target = 0; target < 2; target++) {
        double2* dst = target == 0 ? local : peer;
        const char* where = target == 0 ? "local HBM" : "peer (NVLink)";
        char name[160];
        snprintf(name, sizeof(name), "%s: st.global 16 B/thread, contiguous (512 B per warp)", where);
        timeit(name, (double)bytes, [&] { st_contig<<<sms * 8, 256>>>(dst, n); });
        snprintf(name, sizeof(name), "%s: row segments of  64 B (4 cols), 256 thr x %d CTAs/SM", where, 2);
        timeit(name, (double)bytes, [&] { st_rows<4><<<sms * 2, 256>>>(dst, rowlen, nrows); });
        for (int cps : {1, 2, 4}) {
            snprintf(name, sizeof(name), "%s: row segments of 128 B (8 cols), 256 thr x %d CTAs/SM", where, cps);
            timeit(name, (double)bytes, [&] { st_rows<8><<<sms * cps, 256>>>(dst, rowlen, nrows); });
        }
        snprintf(name, sizeof(name), "%s: row segments of 256 B (16 cols), 512 thr x 1 CTA/SM", where);
        timeit(name, (double)bytes, [&] { st_rows<16><<<sms, 512>>>(dst, rowlen, nrows); });
        snprintf(name, sizeof(name), "%s: row segments of 256 B (16 cols), 256 thr x 2 CTAs/SM", where);
        timeit(name, (double)bytes, [&] { st_rows<16><<<sms * 2, 256>>>(dst, rowlen, nrows); });
        snprintf(name, sizeof(name), "%s: row segments of 512 B (32 cols), 256 thr x 2 CTAs/SM", where);
        timeit(name, (double)bytes, [&] { st_rows<32><<<sms * 2, 256>>>(dst, rowlen, nrows); });
        CK(cudaFuncSetAttribute(st_bulk<65536>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
        snprintf(name, sizeof(name), "%s: TMA bulk store, 64 KB contiguous chunks, 1 CTA/SM", where);
        timeit(name, (double)bytes, [&] { st_bulk<65536><<<sms, 128, 65536>>>((char*)dst, bytes); });
        snprintf(name, sizeof(name), "%s: TMA bulk store,  8 KB contiguous chunks, 2 CTAs/SM", where);
        timeit(name, (double)bytes, [&] { st_bulk<8192><<<sms * 2, 128, 8192>>>((char*)dst, bytes); });
        for (int seg : {4, 8, 16}) {
            CUtensorMap m;
            cuuint64_t dims[2] = {(cuuint64_t)rowlen * 2, (cuuint64_t)nrows};
            cuuint64_t strides[1] = {(cuuint64_t)rowlen * 16};
            cuuint32_t box[2] = {(cuuint32_t)seg * 2, 256};
            cuuint32_t estr[2] = {1, 1};
            CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, dst, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                             CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) { printf("encode failed %d\n", (int)r); continue; }
            const int smem = seg * 16 * 256;
            CK(cudaFuncSetAttribute(st_tensor, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            snprintf(name, sizeof(name), "%s: TMA tensor store, box %3d B x 256 rows, 2 CTAs/SM", where, seg * 16);
            timeit(name, (double)bytes, [&] { st_tensor<<<sms * 2, 128, smem>>>(m, seg, rowlen, nrows); });
        }
    }
    return 0;
}
