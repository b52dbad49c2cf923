// t0_profile.cu -- where the time of the TMA ring kernels goes at 512^3 fp64 on one GPU: the fused forward t0
// (fft_tma_fused_zy_kernel) and the forward X pass (fft_tma_pass_kernel<TMA_XF>) (developer tool, driven by t0_profile.py,
// which builds it and reads what it writes).
//
// Times, with CUDA events over `reps` launches each, alternating the variants per round, at C = 8 (3 slots of 64 KB) and
// C = 4 (6 slots of 32 KB, two consumer groups):
//   fused_cC    the fused kernel body as the library instantiates it (PROBE = 0), at each lag given
//   twin_cC     its movement-only twin (TMA_MOVE): same tickets, counters, ring, loads, stores and L2 hints, no transform
//   xf_cC       the TMA_XF pass on tma_ring (ring_pass_kernel: mover lane, consumer groups, the library's transform) and
//               xf_twin_cC its twin
//   xf_old_twin fft_tma_pass_kernel<TMA_XF>'s structure without arithmetic: 512 threads, a 3-slot ring of 64 KB tiles,
//               thread 0 issues each store, waits until the previous one has read its slot, then loads
//   fused_lag3_promoP, xf_promoP  fft_tma_fused_zy_kernel<C = 8> at lag 3 and fft_tma_pass_kernel<TMA_XF>, with tensor maps
//               of L2 promotion P (0 none, 1 64 B, 2 128 B, 3 256 B); the library promotes one box row
//   copy        a plain TMA copy of the slab with the same 64 KB tiles and 3-slot ring: one read and one write, no hand-off
//   memcpy      cudaMemcpyAsync of the slab, device to device
// and writes one launch's per-tile %globaltimer stamps (TMA_STAMPS) of each ring kernel (fused and twin at the first lag) to
// OUT/stamps_<name>.bin (uint64, TMA_NSTAMP words per ticket or tile).  Prints one JSON object.
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>
#include <functional>

#include "../dfft_kernels.cuh"
#include "../fft_tma.cuh"

using namespace dfft;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

using S512 = Sched<512, 8, 8, 8, 8>;
constexpr int N = 512, CL = 8, NSLOT_OLD = 3;   // the copy and the old XF structure: 64 KB tiles in a 3-slot ring
using G512 = TmaGeom<S512, double, CL>;

// the TMA_XF pass on tma_ring (mover lane, consumer groups): a static tile order, CTA b takes tiles b, b + grid, ...
template <class S, typename T, int C, int MODE> struct TmaPassWork {
    using G_ = TmaGeom<S, T, C>;
    static constexpr bool PUBLISH = false;
    static constexpr bool IN_LINES = MODE == TMA_Z || MODE == TMA_XB, OUT_LINES = MODE == TMA_Z || MODE == TMA_XF;
    const TmaArgs<T>& A;
    const CUtensorMap* map_in;
    const CUtensorMap* map_out;
    long long mine;   // tiles of this CTA
    __device__ long long tile(unsigned n) const { return (long long)blockIdx.x + (long long)n * gridDim.x; }
    __device__ int next(unsigned n, int* d) const
    {
        if (n >= mine) return TMA_W_END;
        d[0] = 0; d[1] = 0; d[2] = 0; d[3] = (int)tile(n);
        return TMA_W_LOAD;
    }
    __device__ bool dep_met(const int*) const { return true; }
    __device__ void load(unsigned n, const int*, cx<T>* buf, uint64_t* bar) const
    {
        const long long t = tile(n), a = t / A.G;
        const int b = (int)(t - a * A.G);
        if constexpr (IN_LINES) tma_bulk_g2s(buf, A.in + a * A.in_SA + (long long)b * C * S::N, G_::TILE_BYTES, bar);
        else {
#pragma unroll
            for (int r = 0; r < G_::NBOX; r++) {
                if constexpr (MODE == TMA_Y) tma_tensor_g2s_3d(buf + r * G_::ROWS * C, map_in, b * C * 2, r * G_::ROWS, (int)a, bar);
                else tma_tensor_g2s_3d(buf + r * G_::ROWS * C, map_in, b * C * 2, (int)a, r * G_::ROWS, bar);
            }
        }
    }
    __device__ void store(unsigned n, const int*, const cx<T>* buf) const
    {
        const long long t = tile(n), a = t / A.G;
        const int b = (int)(t - a * A.G);
        if constexpr (OUT_LINES) tma_bulk_s2g(A.out + a * A.out_SA + (long long)b * C * S::N, buf, G_::TILE_BYTES);
        else {
#pragma unroll
            for (int r = 0; r < G_::NBOX; r++) {
                if constexpr (MODE == TMA_Y) tma_tensor_s2g_3d(map_out, b * C * 2, r * G_::ROWS, (int)a, buf + r * G_::ROWS * C);
                else tma_tensor_s2g_3d(map_out, b * C * 2, (int)a, r * G_::ROWS, buf + r * G_::ROWS * C);
            }
        }
    }
    __device__ void publish(const int*) const {}
    __device__ void transform(const int*, cx<T>* buf, const cx<T>* lut, int bid, int lt) const
    {
        tma_transform<S, T, MODE, C, G_::NT>(buf, lut, bid, lt, A.inv != 0, A.do_scale != 0, A.scale);
    }
    __device__ void finish() const {}
};

template <class S, typename T, int C, int MODE, int PROBE>
__global__ void __launch_bounds__(TMA_CONSUMERS + 32, 1) ring_pass_kernel(const TmaArgs<T> A, unsigned long long* stamps,
                                                                          const __grid_constant__ CUtensorMap map_in, const __grid_constant__ CUtensorMap map_out)
{
    const long long mine = A.ntiles > blockIdx.x ? (A.ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    TmaPassWork<S, T, C, MODE> w{A, &map_in, &map_out, mine};
    tma_ring<S, T, C, PROBE>(w, A.lut, stamps);
}

__global__ void fill_kernel(cx<double>* a, long long n)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        unsigned h = (unsigned)(i * 2654435761ull) ^ (unsigned)(i >> 21);
        a[i].x = (double)(h & 0xffff) / 65536.0 - 0.5;
        a[i].y = (double)(h >> 16) / 65536.0 - 0.5;
    }
}

// plain TMA copy: the ring of fft_tma_pass_kernel (3 slots of one 64 KB tile, bulk load, bulk store, the load of tile i+2 into
// the slot whose store has been read) with the fused kernel's evict_first hints, and nothing done to the data
__global__ void __launch_bounds__(32, 1) tma_copy_kernel(const cx<double>* src, cx<double>* dst, long long ntiles)
{
    extern __shared__ __align__(128) unsigned char raw[];
    __shared__ __align__(8) uint64_t full[NSLOT_OLD];
    if (threadIdx.x != 0) return;
    for (int i = 0; i < NSLOT_OLD; i++) mbar_init(full + i, 1);
    fence_barrier_init();
    const uint64_t pol = l2_policy_evict_first();
    const long long mine = ntiles > blockIdx.x ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    constexpr uint32_t B = G512::TILE_BYTES;
    auto slot = [&](long long i) { return raw + (size_t)(i % NSLOT_OLD) * B; };
    auto tile = [&](long long i) { return (blockIdx.x + i * gridDim.x) * (long long)(B / sizeof(cx<double>)); };
    auto load = [&](long long i) {
        mbar_expect_tx(full + i % NSLOT_OLD, B);
        tma_bulk_g2s_hint(slot(i), src + tile(i), B, full + i % NSLOT_OLD, pol);
    };
    for (long long i = 0; i < mine && i < NSLOT_OLD - 1; i++) load(i);
    for (long long i = 0; i < mine; i++) {
        mbar_wait(full + i % NSLOT_OLD, (uint32_t)((i / NSLOT_OLD) & 1));
        tma_bulk_s2g_hint(dst + tile(i), slot(i), B, pol);
        tma_commit();
        if (i + NSLOT_OLD - 1 < mine) {
            tma_wait_read<1>();
            load(i + NSLOT_OLD - 1);
        }
    }
    tma_wait_all<0>();
}

// fft_tma_pass_kernel<TMA_XF> minus its arithmetic: 512 threads take each slot as it lands, meet at a barrier, and
// thread 0 stores the tile, waits until the previous store has read its slot and loads tile i + 2 into it
__global__ void __launch_bounds__(512, 1) xf_old_twin_kernel(cx<double>* dst, long long ntiles, int G, long long out_SA,
                                                            const __grid_constant__ CUtensorMap map_in)
{
    extern __shared__ __align__(128) unsigned char raw[];
    __shared__ __align__(8) uint64_t full[NSLOT_OLD];
    constexpr uint32_t B = G512::TILE_BYTES;
    if (threadIdx.x == 0) {
        for (int i = 0; i < NSLOT_OLD; i++) mbar_init(full + i, 1);
        fence_barrier_init();
    }
    __syncthreads();
    const long long mine = ntiles > blockIdx.x ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    auto slot = [&](long long i) { return reinterpret_cast<cx<double>*>(raw + (size_t)(i % NSLOT_OLD) * B); };
    auto ab = [&](long long i, long long& a, int& b) {
        const long long t = blockIdx.x + i * gridDim.x;
        a = t / G; b = (int)(t - a * G);
    };
    auto load = [&](long long i) {
        long long a; int b; ab(i, a, b);
        mbar_expect_tx(full + i % NSLOT_OLD, B);
        for (int r = 0; r < G512::NBOX; r++) tma_tensor_g2s_3d(slot(i) + r * G512::ROWS * CL, &map_in, b * CL * 2, (int)a, r * G512::ROWS, full + i % NSLOT_OLD);
    };
    if (threadIdx.x == 0)
        for (long long i = 0; i < mine && i < NSLOT_OLD - 1; i++) load(i);
    for (long long i = 0; i < mine; i++) {
        mbar_wait(full + i % NSLOT_OLD, (uint32_t)((i / NSLOT_OLD) & 1));
        tma_fence_smem_writes();
        __syncthreads();
        if (threadIdx.x == 0) {
            long long a; int b; ab(i, a, b);
            tma_bulk_s2g(dst + a * out_SA + (long long)b * CL * N, slot(i), B);
            tma_commit();
            if (i + NSLOT_OLD - 1 < mine) {
                tma_wait_read<1>();
                load(i + NSLOT_OLD - 1);
            }
        }
    }
    if (threadIdx.x == 0) tma_wait_all<0>();
}

struct Ctx {
    cx<double> *src, *mid, *dst, *lut;
    unsigned long long *plane_done, *stamps;
    unsigned* ticket;
    unsigned long long epoch = 0;
    alignas(64) unsigned char map8[128], map4[128];     // the intermediate, boxes (C, 256, 1): the fused Y role
    alignas(64) unsigned char xmap8[128], xmap4[128];   // src as the XF input, boxes (C, 1, 256)
    int sms;
    long long planes;
};

template <int C, int PROBE> static void launch_fused(Ctx& c, int lag, bool stamps)
{
    using G_ = TmaGeom<S512, double, C>;
    auto kern = fft_tma_fused_zy_probe_kernel<S512, double, C, PROBE>;
    static bool attr = false;
    if (!attr) { CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_::SMEM)); attr = true; }
    TmaFusedArgs<double> a{};
    a.src = c.src; a.mid = c.mid; a.lut = c.lut; a.stamps = stamps ? c.stamps : nullptr;
    FusedCtl f{};
    f.plane_done = c.plane_done; f.ticket = c.ticket; f.planes = c.planes;
    f.GA = N / C; f.GB = N / C;
    f.target = c.epoch += (unsigned long long)f.GA;
    f.lag = lag;
    kern<<<c.sms, TMA_CONSUMERS + 32, G_::SMEM>>>(a, f, *reinterpret_cast<const CUtensorMap*>(C == 8 ? c.map8 : c.map4));
    CK(cudaGetLastError());
}

// the forward X pass of the slab as x_fwd launches it: src [x][y][z] -> dst [y][z][x]
template <int C, int PROBE> static void launch_xf(Ctx& c, bool stamps)
{
    using G_ = TmaGeom<S512, double, C>;
    auto kern = ring_pass_kernel<S512, double, C, TMA_XF, PROBE>;
    static bool attr = false;
    if (!attr) { CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_::SMEM)); attr = true; }
    TmaArgs<double> t{};
    t.lut = c.lut; t.out = c.dst; t.G = N / C; t.ntiles = (long long)N * t.G; t.out_SA = (long long)N * N;
    static CUtensorMap none{};
    kern<<<c.sms, TMA_CONSUMERS + 32, G_::SMEM>>>(t, stamps ? c.stamps : nullptr, *reinterpret_cast<const CUtensorMap*>(C == 8 ? c.xmap8 : c.xmap4), none);
    CK(cudaGetLastError());
}

// the library's fused t0 (lag 3) and TMA_XF pass with tensor maps of each L2 promotion: 0 none, 1 64 B, 2 128 B, 3 256 B
typedef CUresult (*EncFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                          const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static void enc_promo(unsigned char* map, void* base, int C, int b1, int b2, int pr)
{
    static EncFn fn = nullptr;
    if (!fn) { void* p; cudaDriverEntryPointQueryResult q; CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q)); fn = (EncFn)p; }
    cuuint64_t dims[3] = {(cuuint64_t)N * 2, (cuuint64_t)N, (cuuint64_t)N};
    cuuint64_t strides[2] = {(cuuint64_t)N * 16, (cuuint64_t)N * N * 16};
    cuuint32_t box[3] = {(cuuint32_t)C * 2, (cuuint32_t)b1, (cuuint32_t)b2}, estr[3] = {1, 1, 1};
    const CUtensorMapL2promotion prs[4] = {CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B};
    if (fn((CUtensorMap*)map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, prs[pr], CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) { fprintf(stderr, "encode failed\n"); exit(1); }
}
static void launch_fused_promo(Ctx& c, int pr)
{
    alignas(64) static unsigned char m[4][128];
    static bool made[4] = {};
    if (!made[pr]) { enc_promo(m[pr], c.mid, 8, G512::ROWS, 1, pr); made[pr] = true; }
    auto kern = fft_tma_fused_zy_kernel<S512, double, 8>;
    static bool attr = false;
    if (!attr) { CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G512::SMEM)); attr = true; }
    TmaFusedArgs<double> a{};
    a.src = c.src; a.mid = c.mid; a.lut = c.lut;
    FusedCtl f{};
    f.plane_done = c.plane_done; f.ticket = c.ticket; f.planes = c.planes;
    f.GA = N / 8; f.GB = N / 8;
    f.target = c.epoch += (unsigned long long)f.GA;
    f.lag = 3;
    kern<<<c.sms, TMA_CONSUMERS + 32, G512::SMEM>>>(a, f, *reinterpret_cast<const CUtensorMap*>(m[pr]));
    CK(cudaGetLastError());
}
static void launch_xf_lib(Ctx& c, int pr)
{
    alignas(64) static unsigned char m[4][128];
    static bool made[4] = {};
    if (!made[pr]) { enc_promo(m[pr], c.src, 8, 1, G512::ROWS, pr); made[pr] = true; }
    auto kern = fft_tma_pass_kernel<S512, double, 8, TMA_XF>;
    static bool attr = false;
    if (!attr) { CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G512::PASS_SMEM)); attr = true; }
    TmaArgs<double> t{};
    t.lut = c.lut; t.out = c.dst; t.G = N / 8; t.ntiles = (long long)N * t.G; t.out_SA = (long long)N * N;
    static CUtensorMap none{};
    kern<<<c.sms, G512::NT, G512::PASS_SMEM>>>(t, *reinterpret_cast<const CUtensorMap*>(m[pr]), none);
    CK(cudaGetLastError());
}

static void launch_xf_old_twin(Ctx& c)
{
    const size_t smem = NSLOT_OLD * G512::TILE_BYTES;
    static bool attr = false;
    if (!attr) { CK(cudaFuncSetAttribute(xf_old_twin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
    xf_old_twin_kernel<<<c.sms, 512, smem>>>(c.dst, (long long)N * (N / CL), N / CL, (long long)N * N, *reinterpret_cast<const CUtensorMap*>(c.xmap8));
    CK(cudaGetLastError());
}

static void launch_copy(Ctx& c)
{
    static bool attr = false;
    if (!attr) { CK(cudaFuncSetAttribute(tma_copy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(NSLOT_OLD * G512::TILE_BYTES))); attr = true; }
    const long long ntiles = c.planes * (N / CL);
    tma_copy_kernel<<<c.sms, 32, NSLOT_OLD * G512::TILE_BYTES>>>(c.src, c.dst, ntiles);
    CK(cudaGetLastError());
}

template <class F> static float time_ms(F f, int reps)
{
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    CK(cudaEventRecord(a));
    for (int i = 0; i < reps; i++) f();
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, a, b));
    CK(cudaEventDestroy(a)); CK(cudaEventDestroy(b));
    return ms / reps;
}

int main(int argc, char** argv)
{
    std::string out = ".";
    std::vector<int> lags;
    int reps = 20, rounds = 3;
    for (int i = 1; i < argc; i++) {
        if (!strcmp(argv[i], "--out") && i + 1 < argc) out = argv[++i];
        else if (!strcmp(argv[i], "--lag") && i + 1 < argc) lags.push_back(atoi(argv[++i]));
        else if (!strcmp(argv[i], "--reps") && i + 1 < argc) reps = atoi(argv[++i]);
        else if (!strcmp(argv[i], "--rounds") && i + 1 < argc) rounds = atoi(argv[++i]);
        else { fprintf(stderr, "usage: t0_profile --out DIR [--lag L]... [--reps R] [--rounds K]\n"); return 2; }
    }
    if (lags.empty()) lags.push_back(3);
    Ctx c;
    c.planes = N;
    CK(cudaDeviceGetAttribute(&c.sms, cudaDevAttrMultiProcessorCount, 0));
    const long long elems = (long long)N * N * N;
    const size_t bytes = (size_t)elems * sizeof(cx<double>);
    CK(cudaMalloc(&c.src, bytes)); CK(cudaMalloc(&c.mid, bytes)); CK(cudaMalloc(&c.dst, bytes));
    fill_kernel<<<1024, 256>>>(c.src, elems);
    const int rad[3] = {8, 8, 8};
    std::vector<cx<double>> lut = build_lut<double>(3, rad);
    CK(cudaMalloc(&c.lut, (lut.size() * sizeof(cx<double>) + 15) / 16 * 16));
    CK(cudaMemcpy(c.lut, lut.data(), lut.size() * sizeof(cx<double>), cudaMemcpyHostToDevice));
    CK(cudaMalloc(&c.plane_done, N * sizeof(unsigned long long)));
    CK(cudaMemset(c.plane_done, 0, N * sizeof(unsigned long long)));
    CK(cudaMalloc(&c.ticket, 2 * sizeof(unsigned)));
    CK(cudaMemset(c.ticket, 0, 2 * sizeof(unsigned)));
    const size_t nstamped = (size_t)c.planes * 2 * (N / 4);   // the most tickets of any variant (fused at C = 4)
    CK(cudaMalloc(&c.stamps, nstamped * TMA_NSTAMP * sizeof(unsigned long long)));
    const bool maps_ok = tma_encode_3d(c.map8, c.mid, 0, N, N, c.planes, N, (long long)N * N, 8, G512::ROWS, 1) == 0 &&
                         tma_encode_3d(c.map4, c.mid, 0, N, N, c.planes, N, (long long)N * N, 4, G512::ROWS, 1) == 0 &&
                         tma_encode_3d(c.xmap8, c.src, 0, N, N, N, N, (long long)N * N, 8, 1, G512::ROWS) == 0 &&
                         tma_encode_3d(c.xmap4, c.src, 0, N, N, N, N, (long long)N * N, 4, 1, G512::ROWS) == 0;
    if (!maps_ok) { fprintf(stderr, "tensor map encode failed\n"); return 1; }

    struct Variant { std::string name; std::function<void()> run; };
    std::vector<Variant> vs;
    for (int lag : lags) {
        const std::string l = "_lag" + std::to_string(lag);
        vs.push_back({"fused_c8" + l, [&c, lag] { launch_fused<8, 0>(c, lag, false); }});
        vs.push_back({"twin_c8" + l, [&c, lag] { launch_fused<8, TMA_MOVE>(c, lag, false); }});
        vs.push_back({"fused_c4" + l, [&c, lag] { launch_fused<4, 0>(c, lag, false); }});
        vs.push_back({"twin_c4" + l, [&c, lag] { launch_fused<4, TMA_MOVE>(c, lag, false); }});
    }
    vs.push_back({"xf_c8", [&c] { launch_xf<8, 0>(c, false); }});
    vs.push_back({"xf_twin_c8", [&c] { launch_xf<8, TMA_MOVE>(c, false); }});
    vs.push_back({"xf_c4", [&c] { launch_xf<4, 0>(c, false); }});
    vs.push_back({"xf_twin_c4", [&c] { launch_xf<4, TMA_MOVE>(c, false); }});
    vs.push_back({"xf_old_twin", [&c] { launch_xf_old_twin(c); }});
    for (int pr = 0; pr < 4; pr++) {
        vs.push_back({"fused_lag3_promo" + std::to_string(pr), [&c, pr] { launch_fused_promo(c, pr); }});
        vs.push_back({"xf_promo" + std::to_string(pr), [&c, pr] { launch_xf_lib(c, pr); }});
    }
    vs.push_back({"copy", [&c] { launch_copy(c); }});
    vs.push_back({"memcpy", [&c, bytes] { CK(cudaMemcpyAsync(c.dst, c.src, bytes, cudaMemcpyDeviceToDevice)); }});

    for (auto& v : vs) v.run();   // warm-up: every variant once
    CK(cudaDeviceSynchronize());
    printf("{\"sms\": %d, \"reps\": %d, \"rounds\": [", c.sms, reps);
    for (int r = 0; r < rounds; r++) {
        printf("%s{", r ? ", " : "");
        for (size_t k = 0; k < vs.size(); k++) printf("%s\"%s\": %.4f", k ? ", " : "", vs[k].name.c_str(), time_ms(vs[k].run, reps));
        printf("}");
        fflush(stdout);
    }
    printf("]");

    // one stamped launch of each ring kernel, after a stamped warm-up
    printf(", \"stamped\": [");
    bool first = true;
    auto dump = [&](const char* name, size_t tickets, std::function<void()> f) {
        f();
        CK(cudaMemset(c.stamps, 0, nstamped * TMA_NSTAMP * sizeof(unsigned long long)));
        const float ms = time_ms(f, 1);
        std::vector<unsigned long long> h(tickets * TMA_NSTAMP);
        CK(cudaMemcpy(h.data(), c.stamps, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        const std::string path = out + "/stamps_" + name + ".bin";
        FILE* fp = fopen(path.c_str(), "wb");
        if (!fp || fwrite(h.data(), sizeof(unsigned long long), h.size(), fp) != h.size()) { fprintf(stderr, "cannot write %s\n", path.c_str()); exit(1); }
        fclose(fp);
        printf("%s{\"name\": \"%s\", \"ms\": %.4f, \"tickets\": %zu}", first ? "" : ", ", name, ms, tickets);
        first = false;
    };
    const int lag = lags[0];
    const size_t f8 = (size_t)c.planes * 2 * (N / 8), f4 = (size_t)c.planes * 2 * (N / 4);
    dump("fused_c8", f8, [&] { launch_fused<8, TMA_STAMPS>(c, lag, true); });
    dump("twin_c8", f8, [&] { launch_fused<8, TMA_MOVE | TMA_STAMPS>(c, lag, true); });
    dump("fused_c4", f4, [&] { launch_fused<4, TMA_STAMPS>(c, lag, true); });
    dump("twin_c4", f4, [&] { launch_fused<4, TMA_MOVE | TMA_STAMPS>(c, lag, true); });
    dump("xf_c8", (size_t)N * (N / 8), [&] { launch_xf<8, TMA_STAMPS>(c, true); });
    dump("xf_c4", (size_t)N * (N / 4), [&] { launch_xf<4, TMA_STAMPS>(c, true); });
    printf("], \"stamp_lag\": %d, \"nstamp\": %d}\n", lag, (int)TMA_NSTAMP);
    CK(cudaDeviceSynchronize());
    return 0;
}
