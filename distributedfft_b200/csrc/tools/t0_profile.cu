// t0_profile.cu -- where the time of the fused forward t0 (fft_tma_fused_zy_kernel, 512^3 fp64 on one GPU) goes (developer tool,
// driven by t0_profile.py, which builds it and reads what it writes).
//
// Times, with CUDA events over `reps` launches each, alternating the variants per round:
//   fused   the kernel body as the library instantiates it (PROBE = 0), at each lag given
//   twin    the movement-only twin (FZY_MOVE): same tickets, counters, ring, loads, stores and L2 hints, no transform
//   copy    a plain TMA copy of the slab with the same 64 KB tiles and 3-slot ring: one read and one write, no hand-off
//   memcpy  cudaMemcpyAsync of the slab, device to device
// and writes one launch's per-tile %globaltimer stamps (FZY_STAMPS) of the kernel and of the twin at the first lag to
// OUT/stamps_fused.bin and OUT/stamps_twin.bin (uint64, FZY_NSTAMP words per ticket).  Prints one JSON object.
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>

#include "../dfft_kernels.cuh"
#include "../fft_tma.cuh"

using namespace dfft;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

using S512 = Sched<512, 8, 8, 8, 8>;
constexpr int N = 512, CL = 8;
using G512 = TmaGeom<S512, double, CL>;

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
    __shared__ __align__(8) uint64_t full[TMA_NSLOT];
    if (threadIdx.x != 0) return;
    for (int i = 0; i < TMA_NSLOT; i++) mbar_init(full + i, 1);
    fence_barrier_init();
    const uint64_t pol = l2_policy_evict_first();
    const long long mine = ntiles > blockIdx.x ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    constexpr uint32_t B = G512::TILE_BYTES;
    auto slot = [&](long long i) { return raw + (size_t)(i % TMA_NSLOT) * B; };
    auto tile = [&](long long i) { return (blockIdx.x + i * gridDim.x) * (long long)(B / sizeof(cx<double>)); };
    auto load = [&](long long i) {
        mbar_expect_tx(full + i % TMA_NSLOT, B);
        tma_bulk_g2s_hint(slot(i), src + tile(i), B, full + i % TMA_NSLOT, pol);
    };
    for (long long i = 0; i < mine && i < TMA_NSLOT - 1; i++) load(i);
    for (long long i = 0; i < mine; i++) {
        mbar_wait(full + i % TMA_NSLOT, (uint32_t)((i / TMA_NSLOT) & 1));
        tma_bulk_s2g_hint(dst + tile(i), slot(i), B, pol);
        tma_commit();
        if (i + TMA_NSLOT - 1 < mine) {
            tma_wait_read<1>();
            load(i + TMA_NSLOT - 1);
        }
    }
    tma_wait_all<0>();
}

struct Ctx {
    cx<double> *src, *mid, *dst, *lut;
    unsigned long long *plane_done, *stamps;
    unsigned* ticket;
    unsigned long long epoch = 0;
    alignas(64) unsigned char map[128];
    int sms;
    long long planes;
};

template <int PROBE> static void launch_fused(Ctx& c, int lag, bool stamps)
{
    auto kern = fft_tma_fused_zy_probe_kernel<S512, double, CL, PROBE>;
    static bool attr = false;
    if (!attr) { CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G512::SMEM)); attr = true; }
    TmaFusedArgs<double> a{};
    a.src = c.src; a.mid = c.mid; a.lut = c.lut; a.stamps = stamps ? c.stamps : nullptr;
    FusedCtl f{};
    f.plane_done = c.plane_done; f.ticket = c.ticket; f.planes = c.planes;
    f.GA = N / CL; f.GB = N / CL;
    f.target = c.epoch += (unsigned long long)f.GA;
    f.lag = lag;
    kern<<<c.sms, G512::NT + 32, G512::SMEM>>>(a, f, *reinterpret_cast<const CUtensorMap*>(c.map));
    CK(cudaGetLastError());
}

static void launch_copy(Ctx& c)
{
    static bool attr = false;
    if (!attr) { CK(cudaFuncSetAttribute(tma_copy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(TMA_NSLOT * G512::TILE_BYTES))); attr = true; }
    const long long ntiles = c.planes * (N / CL);
    tma_copy_kernel<<<c.sms, 32, TMA_NSLOT * G512::TILE_BYTES>>>(c.src, c.dst, ntiles);
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
    if (lags.empty()) lags.push_back(4);
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
    const size_t ntickets = (size_t)c.planes * 2 * (N / CL);
    CK(cudaMalloc(&c.stamps, ntickets * FZY_NSTAMP * sizeof(unsigned long long)));
    if (tma_encode_3d(c.map, c.mid, 0, N, N, c.planes, N, (long long)N * N, CL, G512::ROWS, 1) != 0) { fprintf(stderr, "tensor map encode failed\n"); return 1; }

    // warm-up: every variant once
    for (int lag : lags) { launch_fused<0>(c, lag, false); launch_fused<FZY_MOVE>(c, lag, false); }
    launch_copy(c);
    CK(cudaMemcpyAsync(c.dst, c.src, bytes, cudaMemcpyDeviceToDevice));
    CK(cudaDeviceSynchronize());

    printf("{\"sms\": %d, \"reps\": %d, \"rounds\": [", c.sms, reps);
    for (int r = 0; r < rounds; r++) {
        printf("%s{", r ? ", " : "");
        for (int lag : lags) {
            printf("\"fused_lag%d\": %.4f, ", lag, time_ms([&] { launch_fused<0>(c, lag, false); }, reps));
            printf("\"twin_lag%d\": %.4f, ", lag, time_ms([&] { launch_fused<FZY_MOVE>(c, lag, false); }, reps));
        }
        printf("\"copy\": %.4f, ", time_ms([&] { launch_copy(c); }, reps));
        printf("\"memcpy\": %.4f}", time_ms([&] { CK(cudaMemcpyAsync(c.dst, c.src, bytes, cudaMemcpyDeviceToDevice)); }, reps));
        fflush(stdout);
    }
    printf("]");

    // one stamped launch of each, after a stamped warm-up
    auto dump = [&](const char* name, float ms) {
        std::vector<unsigned long long> h(ntickets * FZY_NSTAMP);
        CK(cudaMemcpy(h.data(), c.stamps, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        const std::string path = out + "/stamps_" + name + ".bin";
        FILE* f = fopen(path.c_str(), "wb");
        if (!f || fwrite(h.data(), sizeof(unsigned long long), h.size(), f) != h.size()) { fprintf(stderr, "cannot write %s\n", path.c_str()); exit(1); }
        fclose(f);
        printf(", \"stamped_%s_ms\": %.4f", name, ms);
    };
    launch_fused<FZY_STAMPS>(c, lags[0], true);
    CK(cudaMemset(c.stamps, 0, ntickets * FZY_NSTAMP * sizeof(unsigned long long)));
    dump("fused", time_ms([&] { launch_fused<FZY_STAMPS>(c, lags[0], true); }, 1));
    launch_fused<FZY_MOVE | FZY_STAMPS>(c, lags[0], true);
    CK(cudaMemset(c.stamps, 0, ntickets * FZY_NSTAMP * sizeof(unsigned long long)));
    dump("twin", time_ms([&] { launch_fused<FZY_MOVE | FZY_STAMPS>(c, lags[0], true); }, 1));
    printf(", \"stamp_lag\": %d, \"tickets\": %zu, \"nstamp\": %d}\n", lags[0], ntickets, (int)FZY_NSTAMP);
    CK(cudaDeviceSynchronize());
    return 0;
}
