// fft_tma.cuh -- TMA-pipelined pass kernels (sm_90a): the same axis passes as fft_tile_kernel, with the data movement
// handed to the Tensor Memory Accelerator.
//
// One CTA per SM owns a 3-slot shared-memory ring of tiles (C lines x N points, <= 72 KB).  A tile is fetched by TMA
// (one 1-D bulk copy for C contiguous lines, 3-D tensor copies of <= 256 rows for C columns), transformed IN PLACE in its
// slot by S::T * C threads (the Stockham exchanges go through the slot itself: XOR-swizzled inside a line for the
// line-major thread map, row-interleaved for the column-major one), and written back by a TMA store.  While tile i is
// being transformed, tile i+1 is landing and tile i-1 is draining, so global-memory latency never sits on the compute
// threads and no registers are spent on staging.  Which passes use it is chosen per length (dfft_kernels_tma.cu).
//
// What it replaces in the reference: the same generated FFT_main kernels as fft_tile_kernel (templateFFT.cpp:4699-4996);
// X modes also fold the 201 / 120 transposes (fast_transpose/kernels_201.cpp:46-57, kernels_120.cpp:45-57) into the tile.
//
// Modes (tile coordinates (a, b): b = group of C adjacent z columns / C adjacent lines, a = everything slower):
//   TMA_Z  lines   -> lines     dense in, dense out            t0 axis-0 (and its inverse)
//   TMA_Y  columns -> columns   3-D tensor in/out, box (C, rows, 1): transform axis = tensor dim 1      t0 axis-1
//   TMA_XF columns -> lines     3-D tensor in,  box (C, 1, rows): transform axis = tensor dim 2; dense out     t3 forward
//   TMA_XB lines   -> columns   dense in; 3-D tensor out, box (C, 1, rows)                                     t3 backward
#pragma once
#include <cuda.h>

#include "fft_core.cuh"

namespace dfft {

enum { TMA_Z = 0, TMA_Y = 1, TMA_XF = 2, TMA_XB = 3 };
constexpr int TMA_NSLOT = 3;

template <typename T> struct TmaArgs {
    const cx<T>* in;          // dense side (TMA_Z, TMA_XB): tile (a, b) starts at in + a * in_SA + b * C * N
    cx<T>* out;               // dense side (TMA_Z, TMA_XF): tile (a, b) starts at out + a * out_SA + b * C * N
    const cx<T>* lut;
    long long in_SA, out_SA;
    long long ntiles;
    int G;                    // tiles per a
    int inv, do_scale;
    T scale;
};

// ---- PTX ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_bulk_s2g(void* dst, const void* src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_tensor_g2s_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_tensor_s2g_3d(const CUtensorMap* map, int c0, int c1, int c2, const void* src)
{
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];"
                 ::"l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(src)) : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int NLEFT> __device__ __forceinline__ void tma_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(NLEFT) : "memory"); }
template <int NLEFT> __device__ __forceinline__ void tma_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(NLEFT) : "memory"); }
__device__ __forceinline__ void tma_fence_smem_writes() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- slot layouts ---------------------------------------------------------------------------------------------------------
// LAY_LINE : [c][pos], natural (what a bulk copy of C lines delivers / expects)
// LAY_LINES: [c][pos ^ f(pos)], the exchange layout of the line-major thread map (stride-RAD scatters hit distinct banks)
// LAY_COL  : [pos][c], natural (what the tensor copies of C columns deliver / expect); conflict free for the column-major map
// LAY_COLX : [pos][c ^ (pos mod C)], the exchange in which the thread map changes between column-major and line-major
enum { LAY_LINE = 0, LAY_LINES = 1, LAY_COL = 2, LAY_COLX = 3 };
template <int LAY, int N, int C> __device__ __forceinline__ int tma_idx(int c, int pos)
{
    if constexpr (LAY == LAY_LINE) return c * N + pos;
    else if constexpr (LAY == LAY_LINES) return c * N + (pos ^ ((pos >> 3) & 7));
    else if constexpr (LAY == LAY_COL) return pos * C + c;
    else return pos * C + (c ^ (pos & (C - 1)));
}

template <class S, int s, typename T, int LAY, int C, int NT>
__device__ __forceinline__ void tma_exchange(cx<T>* v, cx<T>* buf, int t_w, int c_w, int t_r, int c_r)
{
    constexpr int RAD = S::rad(s), NS = S::ns(s), NB = S::R / RAD;
#pragma unroll
    for (int i = 0; i < NB; i++) {
        const int j = t_w + i * S::T;
        const int k = j % NS;
        const int j0 = (j - k) * RAD + k;
#pragma unroll
        for (int m = 0; m < RAD; m++) buf[tma_idx<LAY, S::N, C>(c_w, j0 + m * NS)] = v[i + m * NB];
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < S::R; u++) v[u] = buf[tma_idx<LAY, S::N, C>(c_r, t_r + u * S::T)];
}

template <class S, int s, typename T, int MODE, int C, int NT> struct TmaStages {
    static constexpr int LAST = S::NSTAGES - 1;
    static __device__ __forceinline__ void run(cx<T>* v, cx<T>* buf, const cx<T>* lut, int t_in, int c_in, int t_out, int c_out)
    {
        stage_compute<S, s, T, false>(v, s == LAST ? t_out : t_in, lut, nullptr);
        __syncthreads();   // s == 0: every thread has read its inputs; s > 0: all gathers of the previous exchange are done
        if constexpr (s < LAST) {
            constexpr bool SWITCH = (MODE == TMA_XF || MODE == TMA_XB) && s + 1 == LAST;   // the thread map changes here
            constexpr int LAY = SWITCH ? LAY_COLX : ((MODE == TMA_Z || MODE == TMA_XB) ? LAY_LINES : LAY_COL);
            if constexpr (SWITCH) tma_exchange<S, s, T, LAY, C, NT>(v, buf, t_in, c_in, t_out, c_out);
            else tma_exchange<S, s, T, LAY, C, NT>(v, buf, t_in, c_in, t_in, c_in);
            TmaStages<S, s + 1, T, MODE, C, NT>::run(v, buf, lut, t_in, c_in, t_out, c_out);
        }
    }
};

template <class S, typename T, int C> struct TmaGeom {
    static constexpr int N = S::N, NT = S::T * C;
    static constexpr int ROWS = N < 256 ? N : 256;            // rows per tensor copy (box limit 256)
    static constexpr int NBOX = N / ROWS;
    static constexpr uint32_t TILE_BYTES = (uint32_t)(N * C * sizeof(cx<T>));
    static constexpr size_t LUT_BYTES = (size_t)((S::lut_size() * sizeof(cx<T>) + 127) / 128 * 128);
    static constexpr size_t SMEM = (size_t)TMA_NSLOT * TILE_BYTES + LUT_BYTES + 128;
    static_assert(N % ROWS == 0, "transform length must be a multiple of the tensor box height");
    static_assert((C & (C - 1)) == 0, "C must be a power of two");
    static_assert(TILE_BYTES % 128 == 0 && SMEM <= 227 * 1024, "tile too large for a 3-slot ring");
    static_assert(S::NSTAGES >= 2, "the map switch of the X modes needs an exchange");
};

template <class S, typename T, int C, int MODE>
__global__ void __launch_bounds__(S::T* C, 1) fft_tma_pass_kernel(const TmaArgs<T> A, const __grid_constant__ CUtensorMap map_in, const __grid_constant__ CUtensorMap map_out)
{
    using G_ = TmaGeom<S, T, C>;
    constexpr int N = S::N, NT = G_::NT, TT = S::T, ROWS = G_::ROWS, NBOX = G_::NBOX;
    constexpr bool IN_LINES = MODE == TMA_Z || MODE == TMA_XB, OUT_LINES = MODE == TMA_Z || MODE == TMA_XF;
    extern __shared__ __align__(128) unsigned char tma_raw[];
    cx<T>* const lut_s = reinterpret_cast<cx<T>*>(tma_raw + (size_t)TMA_NSLOT * G_::TILE_BYTES);
    uint64_t* const full = reinterpret_cast<uint64_t*>(tma_raw + (size_t)TMA_NSLOT * G_::TILE_BYTES + G_::LUT_BYTES);
    auto slot = [&](int i) { return reinterpret_cast<cx<T>*>(tma_raw + (size_t)i * G_::TILE_BYTES); };
    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int i = 0; i < TMA_NSLOT; i++) mbar_init(full + i, 1);
        fence_barrier_init();
    }
    for (int i = tid; i < S::lut_size(); i += NT) lut_s[i] = A.lut[i];
    __syncthreads();
    // thread maps: line-major (t fastest) on the dense side, column-major (c fastest) on the tensor side
    const int t_in = IN_LINES ? tid % TT : tid / C, c_in = IN_LINES ? tid / TT : tid % C;
    const int t_out = OUT_LINES ? tid % TT : tid / C, c_out = OUT_LINES ? tid / TT : tid % C;
    const long long mine = A.ntiles > blockIdx.x ? (A.ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    auto load = [&](long long i) {   // thread 0
        const int s = (int)(i % TMA_NSLOT);
        const long long tile = (long long)blockIdx.x + i * gridDim.x;
        const long long a = tile / A.G;
        const int b = (int)(tile - a * A.G);
        mbar_expect_tx(full + s, G_::TILE_BYTES);
        if constexpr (IN_LINES) tma_bulk_g2s(slot(s), A.in + a * A.in_SA + (long long)b * C * N, G_::TILE_BYTES, full + s);
        else {
#pragma unroll
            for (int r = 0; r < NBOX; r++) {
                if constexpr (MODE == TMA_Y) tma_tensor_g2s_3d(slot(s) + r * ROWS * C, &map_in, b * C * 2, r * ROWS, (int)a, full + s);
                else tma_tensor_g2s_3d(slot(s) + r * ROWS * C, &map_in, b * C * 2, (int)a, r * ROWS, full + s);
            }
        }
    };
    if (tid == 0)
        for (long long i = 0; i < mine && i < TMA_NSLOT - 1; i++) load(i);
    for (long long i = 0; i < mine; i++) {
        const int s = (int)(i % TMA_NSLOT);
        cx<T>* buf = slot(s);
        mbar_wait(full + s, (uint32_t)((i / TMA_NSLOT) & 1));
        cx<T> v[S::R];
#pragma unroll
        for (int u = 0; u < S::R; u++) v[u] = buf[tma_idx<IN_LINES ? LAY_LINE : LAY_COL, N, C>(c_in, t_in + u * TT)];
        if (A.inv) {
#pragma unroll
            for (int u = 0; u < S::R; u++) v[u] = cswap(v[u]);
        }
        TmaStages<S, 0, T, MODE, C, NT>::run(v, buf, lut_s, t_in, c_in, t_out, c_out);
        if (A.inv) {
#pragma unroll
            for (int u = 0; u < S::R; u++) v[u] = cswap(v[u]);
        }
        if (A.do_scale) {
#pragma unroll
            for (int u = 0; u < S::R; u++) { v[u].x *= A.scale; v[u].y *= A.scale; }
        }
#pragma unroll
        for (int u = 0; u < S::R; u++) buf[tma_idx<OUT_LINES ? LAY_LINE : LAY_COL, N, C>(c_out, t_out + u * TT)] = v[u];
        tma_fence_smem_writes();        // generic-proxy writes -> visible to the TMA store
        __syncthreads();
        if (tid == 0) {
            const long long tile = (long long)blockIdx.x + i * gridDim.x;
            const long long a = tile / A.G;
            const int b = (int)(tile - a * A.G);
            if constexpr (OUT_LINES) tma_bulk_s2g(A.out + a * A.out_SA + (long long)b * C * N, buf, G_::TILE_BYTES);
            else {
#pragma unroll
                for (int r = 0; r < NBOX; r++) {
                    if constexpr (MODE == TMA_Y) tma_tensor_s2g_3d(&map_out, b * C * 2, r * ROWS, (int)a, buf + r * ROWS * C);
                    else tma_tensor_s2g_3d(&map_out, b * C * 2, (int)a, r * ROWS, buf + r * ROWS * C);
                }
            }
            tma_commit();
            if (i + TMA_NSLOT - 1 < mine) {
                tma_wait_read<1>();     // the store of tile i-1 has drained its slot, which tile i+2 reuses
                load(i + TMA_NSLOT - 1);
            }
        }
    }
    if (tid == 0) tma_wait_all<0>();
}

}  // namespace dfft
