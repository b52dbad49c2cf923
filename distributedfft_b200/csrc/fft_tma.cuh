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
#include "fft_passes.cuh"

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

// CTA-wide barrier of the threads that transform a tile: the whole CTA in the pass kernels; in the fused kernel, whose
// mover warp has left the loop, the NT consumer threads on named barrier 1
template <bool CONS, int NT> __device__ __forceinline__ void tma_sync()
{
    if constexpr (CONS) asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory");
    else __syncthreads();
}

template <class S, int s, typename T, int LAY, int C, int NT, bool CONS = false>
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
    tma_sync<CONS, NT>();
#pragma unroll
    for (int u = 0; u < S::R; u++) v[u] = buf[tma_idx<LAY, S::N, C>(c_r, t_r + u * S::T)];
}

template <class S, int s, typename T, int MODE, int C, int NT, bool CONS = false> struct TmaStages {
    static constexpr int LAST = S::NSTAGES - 1;
    static __device__ __forceinline__ void run(cx<T>* v, cx<T>* buf, const cx<T>* lut, int t_in, int c_in, int t_out, int c_out)
    {
        stage_compute<S, s, T, false>(v, s == LAST ? t_out : t_in, lut, nullptr);
        tma_sync<CONS, NT>();   // s == 0: every thread has read its inputs; s > 0: all gathers of the previous exchange are done
        if constexpr (s < LAST) {
            constexpr bool SWITCH = (MODE == TMA_XF || MODE == TMA_XB) && s + 1 == LAST;   // the thread map changes here
            constexpr int LAY = SWITCH ? LAY_COLX : ((MODE == TMA_Z || MODE == TMA_XB) ? LAY_LINES : LAY_COL);
            if constexpr (SWITCH) tma_exchange<S, s, T, LAY, C, NT, CONS>(v, buf, t_in, c_in, t_out, c_out);
            else tma_exchange<S, s, T, LAY, C, NT, CONS>(v, buf, t_in, c_in, t_in, c_in);
            TmaStages<S, s + 1, T, MODE, C, NT, CONS>::run(v, buf, lut, t_in, c_in, t_out, c_out);
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

// ---- forward t0 in one kernel: the Z pass and the natural Y pass of square planes, intermediate resident in L2 -------------
// The two-sweep t0 reads and writes the slab twice through DRAM; here a plane's Z output is consumed by its Y tiles while it
// is still in L2, so t0 costs one DRAM read and one DRAM write of the slab.  Work comes from the ticket order of
// fft_fused2_kernel (fused2_decode: Z runs `lag` planes ahead of Y) and the same monotonic per-plane counters.
//   Z role: src -> mid, C contiguous lines per tile, 1-D bulk copies (TMA_Z's tile and thread map)
//   Y role: mid -> mid in place, C columns per tile, 3-D tensor copies through map_mid (TMA_Y's tile, map and thread map)
// The CTA is NT consumer threads and one mover warp, of which one lane works.  The consumers only transform: they take the
// slots in ring order as they land (mbarrier `full`) and hand each back (mbarrier `done`).  The mover does all the rest in
// one polling loop that never blocks on anything but its own bulk groups:
//   - a handed-back tile: issue its store, wait until the store has READ the slot (cp.async.bulk.wait_group.read) and
//     count the slot free; a Z tile's store stays pending, and is published (plane counter += 1) as soon as the mover has
//     nothing else to do (wait_group 0), or when a later store has been issued and everything older is complete (wait_group 1);
//   - a free slot: draw a ticket and issue its load -- a Y tile's only after its plane's counter has reached the target,
//     polled, so that a Y tile waiting for its plane holds up neither the stores nor the publications of this CTA;
// Why a mover (csrc/tools/t0_profile.py, DESIGN.md 3.4): when consumer thread 0 issued the stores, it waited for the
// previous store's completion before every tile, and each slot stayed held until its store was complete; at 512^3 fp64 the
// transform itself then took less than half of the time per tile.  Here the consumers never wait for a store, and a slot
// is refilled as soon as its store has read it.
// Deadlock freedom, whatever the residency: a Y ticket waits only for Z tickets of its plane, and all of them are lower.
// Each of those was drawn by a running mover with a free slot, so its load is in flight; the tiles ahead of it in that CTA's
// ring have still lower tickets (tickets rise per CTA), so by induction they land, and the consumers, who wait for nothing
// but landed slots, hand them back in order.  The Z tile's store is then issued, and it is published without waiting for a
// later tile to land: the mover publishes it the first time it finds nothing else to do, which it must while the next
// ticket is a Y tile still waiting for its plane (perhaps for exactly this tile), and at the latest with the next store.
// Proxy order of the hand-over: consumers' smem writes, fence.proxy.async.shared::cta, named barrier, `done` arrive; the
// mover's mbarrier test_wait, then its TMA store.  Z tile: store's wait_group, fence.proxy.async, __threadfence, counter add;
// Y tile: ld.acquire.gpu of the counter, fence.proxy.async, tensor load.
// L2 policy per instruction (createpolicy): the slab is read once and the finished Y columns are not read again by this
// kernel, so the Z loads and the Y stores are evict_first; the Z stores of the intermediate are evict_last, so that they
// survive until their Y tiles read them.  At 512^3 fp64 on H100 the three hints together take t0 from 2.90 to 2.30 ms at
// lag 4 (DESIGN.md 3.4).  No persisting-L2 carve-out is used: that is a device-wide setting.
template <typename T> struct TmaFusedArgs {
    const cx<T>* src;    // Z role input (dense planes of N x N)
    cx<T>* mid;          // Z role output, Y role input and output (described by map_mid)
    const cx<T>* lut;
    unsigned long long* stamps;   // FZY_STAMPS instantiations only: FZY_NSTAMP words per ticket; null in the library
};

// Measurement instantiations of fft_tma_fused_zy_kernel (PROBE bits; the library instantiates PROBE = 0 only, and
// csrc/tools/t0_profile.py builds the others):
//   FZY_MOVE   the movement-only twin: same tickets, plane counters, ring, loads, stores and L2 hints, but the consumers copy
//              the slot through unchanged (no butterflies, no exchanges) -- its time is what the ring, the hand-off through
//              the plane counters and the L2 traffic allow without any arithmetic
//   FZY_STAMPS %globaltimer stamps per tile into A.stamps[ticket * FZY_NSTAMP + field], fields FZS_*
enum { FZY_MOVE = 1, FZY_STAMPS = 2 };
enum { FZS_WHO = 0,        // blockIdx.x * 2 + (Y tile ? 1 : 0)
       FZS_TICKET,         // mover: ticket drawn
       FZS_DEP,            // mover: plane counter satisfied (a Z tile: = FZS_TICKET)
       FZS_LOAD,           // mover: load issued
       FZS_READY,          // consumer thread 0: done with the previous tile, starts waiting for this slot
       FZS_FULL,           // consumer thread 0: slot full
       FZS_DONE,           // consumer thread 0: transform done (after the consumers' barrier), tile handed to the mover
       FZS_STORE,          // mover: store issued
       FZS_FREED,          // mover: the store has read the slot, slot freed
       FZS_RETIRED,        // mover: a Z tile's store is complete and the tile published (a Y tile: just after FZS_FREED)
       FZY_NSTAMP };

__device__ __forceinline__ uint64_t l2_policy_evict_first()
{
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last()
{
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void tma_bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ void tma_bulk_s2g_hint(void* dst, const void* src, uint32_t bytes, uint64_t pol)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes), "l"(pol) : "memory");
}
__device__ __forceinline__ void tma_tensor_s2g_3d_hint(const CUtensorMap* map, int c0, int c1, int c2, const void* src, uint64_t pol)
{
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%1, %2, %3}], [%4], %5;"
                 ::"l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(src)), "l"(pol) : "memory");
}

__device__ __forceinline__ void tma_mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// non-blocking test of a phase (mbarrier.try_wait may suspend the thread for a while; a thread that polls several things must not)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t phase)
{
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase) : "memory");
    return ok != 0;
}

template <class S, typename T, int C, int PROBE>
__device__ __forceinline__ void tma_fused_zy_body(const TmaFusedArgs<T>& A, const FusedCtl& F, const CUtensorMap* map_mid)
{
    using G_ = TmaGeom<S, T, C>;
    constexpr int N = S::N, NT = G_::NT, TT = S::T, ROWS = G_::ROWS, NBOX = G_::NBOX;
    constexpr bool STAMPS = (PROBE & FZY_STAMPS) != 0;
    extern __shared__ __align__(128) unsigned char tma_raw[];
    cx<T>* const lut_s = reinterpret_cast<cx<T>*>(tma_raw + (size_t)TMA_NSLOT * G_::TILE_BYTES);
    uint64_t* const full = reinterpret_cast<uint64_t*>(tma_raw + (size_t)TMA_NSLOT * G_::TILE_BYTES + G_::LUT_BYTES);
    uint64_t* const done = full + TMA_NSLOT;   // per slot: the consumers have written the tile back into it
    int* const desc = reinterpret_cast<int*>(done + TMA_NSLOT);   // per slot: role (-1 end, 0 Z, 1 Y), plane, tile
    unsigned* const slot_ticket = reinterpret_cast<unsigned*>(desc + 3 * TMA_NSLOT);   // per slot: ticket (FZY_STAMPS only)
    static_assert(2 * TMA_NSLOT * sizeof(uint64_t) + 4 * TMA_NSLOT * sizeof(int) <= 128, "ring control words exceed the reserve");
    auto slot = [&](int i) { return reinterpret_cast<cx<T>*>(tma_raw + (size_t)i * G_::TILE_BYTES); };
    auto stamp = [&](unsigned t, int f) {
        if constexpr (STAMPS) A.stamps[(size_t)t * FZY_NSTAMP + f] = gtime_ns();
    };
    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int i = 0; i < TMA_NSLOT; i++) { mbar_init(full + i, 1); mbar_init(done + i, 1); }
        fence_barrier_init();
    }
    for (int i = tid; i < S::lut_size(); i += NT + 32) lut_s[i] = A.lut[i];
    __syncthreads();
    const Fused2Order o = fused2_prepare(F);

    if (tid >= NT) {
        // ---- mover: one lane draws the tickets, issues every load and store, frees the slots and publishes the Z tiles ----
        if (tid == NT) {
            unsigned n_load = 0;    // ring position of the next ticket
            unsigned n_store = 0;   // ring position of the next tile the consumers hand back; every earlier slot is free
            bool waiting = false;   // the ticket at n_load is a Y tile whose plane is not complete yet
            bool ended = false;     // the end marker is in the ring
            bool pend = false;      // the last store issued is a Z tile's, not yet known complete
            unsigned pend_plane = 0, pend_ticket = 0;
            auto publish = [&]() {   // the pending tile's store is complete
                stamp(pend_ticket, FZS_RETIRED);
                asm volatile("fence.proxy.async;" ::: "memory");
                __threadfence();
                atomicAdd(F.plane_done + pend_plane, 1ull);
                pend = false;
            };
            SpinGuard guard;
            for (;;) {
                bool acted = false;
                // a transformed tile: store it, and free its slot as soon as the store has read it
                const int ss = (int)(n_store % TMA_NSLOT);
                if (n_store < n_load && mbar_test_wait(done + ss, (n_store / TMA_NSLOT) & 1)) {
                    const int role = desc[ss * 3 + 0], plane = desc[ss * 3 + 1], idx = desc[ss * 3 + 2];
                    if (role < 0) break;
                    const unsigned t = STAMPS ? slot_ticket[ss] : 0u;
                    cx<T>* buf = slot(ss);
                    // policies made at the point of use: held across the loop they cost spill slots
                    if (role == 0) tma_bulk_s2g_hint(A.mid + ((long long)plane * o.GA + idx) * (C * N), buf, G_::TILE_BYTES, l2_policy_evict_last());
                    else {
                        const uint64_t write_once = l2_policy_evict_first();
#pragma unroll
                        for (int r = 0; r < NBOX; r++) tma_tensor_s2g_3d_hint(map_mid, idx * C * 2, r * ROWS, plane, buf + r * ROWS * C, write_once);
                    }
                    tma_commit();
                    stamp(t, FZS_STORE);
                    tma_wait_read<0>();
                    stamp(t, FZS_FREED);
                    if (pend) { tma_wait_all<1>(); publish(); }   // the pending tile's store is older than this one: complete
                    if (role == 0) { pend = true; pend_plane = (unsigned)plane; pend_ticket = t; }
                    else stamp(t, FZS_RETIRED);   // nothing waits for a Y tile's completion but the kernel's end
                    n_store++;
                    acted = true;
                }
                // a free slot: draw the next ticket and load its tile (a Y tile once its plane is complete)
                if (!ended && !waiting && n_load < n_store + TMA_NSLOT) {
                    const int s = (int)(n_load % TMA_NSLOT);
                    const unsigned t = atomicAdd(F.ticket, 1u);
                    if (t >= o.total) {   // end marker, no bytes
                        desc[s * 3] = -1;
                        tma_mbar_arrive(full + s);
                        ended = true;
                        n_load++;
                    } else {
                        bool z;
                        unsigned plane, idx;
                        fused2_decode(o, t, z, plane, idx);
                        desc[s * 3 + 0] = z ? 0 : 1; desc[s * 3 + 1] = (int)plane; desc[s * 3 + 2] = (int)idx;
                        if constexpr (STAMPS) {
                            slot_ticket[s] = t;
                            A.stamps[(size_t)t * FZY_NSTAMP + FZS_WHO] = blockIdx.x * 2u + (z ? 0u : 1u);
                            stamp(t, FZS_TICKET);
                        }
                        if (z) {
                            stamp(t, FZS_DEP);
                            mbar_expect_tx(full + s, G_::TILE_BYTES);
                            tma_bulk_g2s_hint(slot(s), A.src + ((long long)plane * o.GA + idx) * (C * N), G_::TILE_BYTES, full + s, l2_policy_evict_first());
                            stamp(t, FZS_LOAD);
                            n_load++;
                        } else waiting = true;
                    }
                    acted = true;
                }
                if (waiting) {   // every Z tile of the plane is stored
                    const int s = (int)(n_load % TMA_NSLOT);
                    unsigned long long v;
                    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(F.plane_done + desc[s * 3 + 1]) : "memory");
                    if (v >= F.target) {
                        asm volatile("fence.proxy.async;" ::: "memory");   // the acquired data is read through the async proxy
                        stamp(slot_ticket[s], FZS_DEP);
                        mbar_expect_tx(full + s, G_::TILE_BYTES);
#pragma unroll
                        for (int r = 0; r < NBOX; r++)
                            tma_tensor_g2s_3d(slot(s) + r * ROWS * C, map_mid, desc[s * 3 + 2] * C * 2, r * ROWS, desc[s * 3 + 1], full + s);
                        stamp(slot_ticket[s], FZS_LOAD);
                        waiting = false;
                        n_load++;
                        acted = true;
                    }
                }
                if (acted) { guard = SpinGuard{}; continue; }
                // nothing to do: publish the pending tile now rather than with the next store, since Y tiles of other CTAs
                // (or the very Y ticket this CTA waits on) may be waiting for it
                if (pend) {
                    tma_wait_all<0>();
                    publish();
                } else {
                    if (waiting) __nanosleep(64);
                    guard.tick();
                }
            }
            tma_wait_all<0>();
            if (pend) publish();
            const unsigned left = atomicAdd(F.ticket + 1, 1u);   // the last CTA to leave re-arms the ticket counter
            if (left == gridDim.x - 1) { F.ticket[0] = 0; F.ticket[1] = 0; __threadfence(); }
        }
        return;
    }

    // ---- consumers: transform the slots in ring order and hand each back to the mover ----
    for (unsigned n = 0;; n++) {
        const int s = (int)(n % TMA_NSLOT);
        unsigned long long ready = 0;
        if constexpr (STAMPS) ready = gtime_ns();
        mbar_wait(full + s, (n / TMA_NSLOT) & 1);
        const int role = desc[s * 3 + 0];
        if (role < 0) {   // end marker: pass it on, so that the mover stops after the last store
            if (tid == 0) tma_mbar_arrive(done + s);
            break;
        }
        if constexpr (STAMPS) {
            if (tid == 0) {
                A.stamps[(size_t)slot_ticket[s] * FZY_NSTAMP + FZS_READY] = ready;
                stamp(slot_ticket[s], FZS_FULL);
            }
        }
        cx<T>* buf = slot(s);
        cx<T> v[S::R];
        if constexpr ((PROBE & FZY_MOVE) != 0) {
            // the twin: the slot leaves as it arrived
        } else if (role == 0) {
            const int t = tid % TT, c = tid / TT;
#pragma unroll
            for (int u = 0; u < S::R; u++) v[u] = buf[tma_idx<LAY_LINE, N, C>(c, t + u * TT)];
            TmaStages<S, 0, T, TMA_Z, C, NT, true>::run(v, buf, lut_s, t, c, t, c);
#pragma unroll
            for (int u = 0; u < S::R; u++) buf[tma_idx<LAY_LINE, N, C>(c, t + u * TT)] = v[u];
        } else {
            const int t = tid / C, c = tid % C;
#pragma unroll
            for (int u = 0; u < S::R; u++) v[u] = buf[tma_idx<LAY_COL, N, C>(c, t + u * TT)];
            TmaStages<S, 0, T, TMA_Y, C, NT, true>::run(v, buf, lut_s, t, c, t, c);
#pragma unroll
            for (int u = 0; u < S::R; u++) buf[tma_idx<LAY_COL, N, C>(c, t + u * TT)] = v[u];
        }
        tma_fence_smem_writes();   // generic-proxy writes -> visible to the mover's TMA store
        tma_sync<true, NT>();
        if (tid == 0) {
            stamp(slot_ticket[s], FZS_DONE);
            tma_mbar_arrive(done + s);
        }
    }
}

template <class S, typename T, int C>
__global__ void __launch_bounds__(S::T* C + 32, 1) fft_tma_fused_zy_kernel(const TmaFusedArgs<T> A, const FusedCtl F,
                                                                            const __grid_constant__ CUtensorMap map_mid)
{
    tma_fused_zy_body<S, T, C, 0>(A, F, &map_mid);
}

// the measurement instantiations (FZY_MOVE, FZY_STAMPS), launched like fft_tma_fused_zy_kernel
template <class S, typename T, int C, int PROBE>
__global__ void __launch_bounds__(S::T* C + 32, 1) fft_tma_fused_zy_probe_kernel(const TmaFusedArgs<T> A, const FusedCtl F,
                                                                                  const __grid_constant__ CUtensorMap map_mid)
{
    tma_fused_zy_body<S, T, C, PROBE>(A, F, &map_mid);
}

}  // namespace dfft
