// fft_tma.cuh -- TMA-pipelined pass kernels (sm_90a): the same axis passes as fft_tile_kernel, with the data movement
// handed to the Tensor Memory Accelerator.
//
// One CTA per SM owns a shared-memory ring of tiles (C lines x N points each).  A tile is fetched by TMA (one 1-D bulk copy
// for C contiguous lines, 3-D tensor copies of <= 256 rows for C columns), transformed IN PLACE in its slot by S::T * C
// threads (the Stockham exchanges go through the slot itself: XOR-swizzled inside a line for the line-major thread map,
// row-interleaved for the column-major one), and written back by a TMA store.  While one tile is being transformed, the
// next is landing and the previous one draining, so no registers are spent on staging.  The pass kernels keep a 3-slot
// ring fed by thread 0; the fused forward t0 runs on tma_ring, whose loads and stores are all issued by a mover lane.
// Which passes use them is chosen per length (dfft_kernels_tma.cu).
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
constexpr int TMA_CONSUMERS = 512;   // tma_ring: consumer threads per CTA; one mover warp comes on top
constexpr int TMA_PASS_NSLOT = 3;    // fft_tma_pass_kernel's ring

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
// wait_group.read takes an immediate: at most `left` (< MAX) of the committed store groups may still be reading shared memory
template <int MAX> __device__ __forceinline__ void tma_wait_read_dyn(int left)
{
    if constexpr (MAX > 1) {
        if (left >= MAX - 1) { tma_wait_read<MAX - 1>(); return; }
        tma_wait_read_dyn<MAX - 1>(left);
    } else tma_wait_read<0>();
}
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

// barrier of the NT consumer threads that transform one tile: named barrier `bid` (1 + their group; 0 is __syncthreads)
template <int NT> __device__ __forceinline__ void tma_sync(int bid) { asm volatile("bar.sync %0, %1;" ::"r"(bid), "n"(NT) : "memory"); }

template <class S, int s, typename T, int LAY, int C, int NT>
__device__ __forceinline__ void tma_exchange(cx<T>* v, cx<T>* buf, int bid, int t_w, int c_w, int t_r, int c_r)
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
    tma_sync<NT>(bid);
#pragma unroll
    for (int u = 0; u < S::R; u++) v[u] = buf[tma_idx<LAY, S::N, C>(c_r, t_r + u * S::T)];
}

template <class S, int s, typename T, int MODE, int C, int NT> struct TmaStages {
    static constexpr int LAST = S::NSTAGES - 1;
    static __device__ __forceinline__ void run(cx<T>* v, cx<T>* buf, const cx<T>* lut, int bid, int t_in, int c_in, int t_out, int c_out)
    {
        stage_compute<S, s, T, false>(v, s == LAST ? t_out : t_in, lut, nullptr);
        tma_sync<NT>(bid);   // s == 0: every thread has read its inputs; s > 0: all gathers of the previous exchange are done
        if constexpr (s < LAST) {
            constexpr bool SWITCH = (MODE == TMA_XF || MODE == TMA_XB) && s + 1 == LAST;   // the thread map changes here
            constexpr int LAY = SWITCH ? LAY_COLX : ((MODE == TMA_Z || MODE == TMA_XB) ? LAY_LINES : LAY_COL);
            if constexpr (SWITCH) tma_exchange<S, s, T, LAY, C, NT>(v, buf, bid, t_in, c_in, t_out, c_out);
            else tma_exchange<S, s, T, LAY, C, NT>(v, buf, bid, t_in, c_in, t_in, c_in);
            TmaStages<S, s + 1, T, MODE, C, NT>::run(v, buf, lut, bid, t_in, c_in, t_out, c_out);
        }
    }
};

// one tile transformed in place by the NT threads of a group: load from the slot in the input layout, the stages, store back
// in the output layout (LAY_LINE on the dense side, LAY_COL on the tensor side)
template <class S, typename T, int MODE, int C, int NT>
__device__ __forceinline__ void tma_transform(cx<T>* buf, const cx<T>* lut, int bid, int lt, bool inv, bool do_scale, T scale)
{
    constexpr int TT = S::T;
    constexpr bool IN_LINES = MODE == TMA_Z || MODE == TMA_XB, OUT_LINES = MODE == TMA_Z || MODE == TMA_XF;
    // thread maps: line-major (t fastest) on the dense side, column-major (c fastest) on the tensor side
    const int t_in = IN_LINES ? lt % TT : lt / C, c_in = IN_LINES ? lt / TT : lt % C;
    const int t_out = OUT_LINES ? lt % TT : lt / C, c_out = OUT_LINES ? lt / TT : lt % C;
    cx<T> v[S::R];
#pragma unroll
    for (int u = 0; u < S::R; u++) v[u] = buf[tma_idx<IN_LINES ? LAY_LINE : LAY_COL, S::N, C>(c_in, t_in + u * TT)];
    if (inv) {
#pragma unroll
        for (int u = 0; u < S::R; u++) v[u] = cswap(v[u]);
    }
    TmaStages<S, 0, T, MODE, C, NT>::run(v, buf, lut, bid, t_in, c_in, t_out, c_out);
    if (inv) {
#pragma unroll
        for (int u = 0; u < S::R; u++) v[u] = cswap(v[u]);
    }
    if (do_scale) {
#pragma unroll
        for (int u = 0; u < S::R; u++) { v[u].x *= scale; v[u].y *= scale; }
    }
#pragma unroll
    for (int u = 0; u < S::R; u++) buf[tma_idx<OUT_LINES ? LAY_LINE : LAY_COL, S::N, C>(c_out, t_out + u * TT)] = v[u];
}

// Shared memory: NSLOT tiles, the twiddles, and per slot the control words (mbarriers `full` and `done`, a 4-int descriptor).
// NSLOT is whatever fits in the 227 KB an SM grants one CTA: 3 slots of 64 KB tiles, 6 of 32 KB tiles.
template <class S, typename T, int C> struct TmaGeom {
    static constexpr int N = S::N, NT = S::T * C;
    static constexpr int NGROUP = TMA_CONSUMERS / NT;          // consumer groups, each transforming its own tile
    static constexpr int ROWS = N < 256 ? N : 256;            // rows per tensor copy (box limit 256)
    static constexpr int NBOX = N / ROWS;
    static constexpr uint32_t TILE_BYTES = (uint32_t)(N * C * sizeof(cx<T>));
    static constexpr size_t LUT_BYTES = (size_t)((S::lut_size() * sizeof(cx<T>) + 127) / 128 * 128);
    static constexpr size_t SMEM_MAX = 227 * 1024;
    static constexpr size_t ctrl_bytes(size_t n) { return (n * (2 * sizeof(uint64_t) + 4 * sizeof(int)) + 127) / 128 * 128; }
    static constexpr int FIT = (int)((SMEM_MAX - LUT_BYTES) / TILE_BYTES);
    static constexpr int NSLOT = FIT * (size_t)TILE_BYTES + LUT_BYTES + ctrl_bytes(FIT) <= SMEM_MAX ? FIT : FIT - 1;
    static constexpr size_t CTRL_BYTES = ctrl_bytes(NSLOT);
    static constexpr size_t SMEM = (size_t)NSLOT * TILE_BYTES + LUT_BYTES + CTRL_BYTES;                 // tma_ring
    static constexpr size_t PASS_SMEM = (size_t)TMA_PASS_NSLOT * TILE_BYTES + LUT_BYTES + 128;          // fft_tma_pass_kernel
    static_assert(N % ROWS == 0, "transform length must be a multiple of the tensor box height");
    static_assert((C & (C - 1)) == 0, "C must be a power of two");
    static_assert(TILE_BYTES % 128 == 0 && PASS_SMEM <= SMEM_MAX, "tile too large for a 3-slot ring");
    static_assert(S::NSTAGES >= 2, "the map switch of the X modes needs an exchange");
};

// Measurement instantiations of the TMA kernels (PROBE bits; the library instantiates PROBE = 0 only, and
// csrc/tools/t0_profile.py builds the others):
//   TMA_MOVE   the movement-only twin: same ring, work order, loads, stores, hand-offs and L2 hints, but the consumers pass
//              the slot through unchanged (no butterflies, no exchanges) -- its time is what the data movement allows
//   TMA_STAMPS %globaltimer stamps per tile into stamps[id * TMA_NSTAMP + field], fields TMS_*; id = the fused kernel's
//              ticket, the pass kernel's tile index
enum { TMA_MOVE = 1, TMA_STAMPS = 2 };
enum { TMS_WHO = 0,        // blockIdx.x * 2 + (fused Y tile ? 1 : 0)
       TMS_TICKET,         // mover: tile drawn
       TMS_DEP,            // mover: plane counter satisfied (otherwise = TMS_TICKET)
       TMS_LOAD,           // mover: load issued
       TMS_READY,          // consumer group: done with its previous tile, starts waiting for this slot
       TMS_FULL,           // consumer group: slot full
       TMS_DONE,           // consumer group: transform done (after the group's barrier), tile handed to the mover
       TMS_STORE,          // mover: store issued
       TMS_FREED,          // mover: the store has read the slot, slot freed
       TMS_RETIRED,        // mover: a fused Z tile's store is complete and the tile published (others: = TMS_FREED)
       TMA_NSTAMP };

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

// ---- the ring: one mover lane, NGROUP consumer groups -----------------------------------------------------------------------
// Ring position n lives in slot n % NSLOT and is transformed by consumer group n % NGROUP; each group takes its positions in
// order as they land (mbarrier `full`) and hands each back (mbarrier `done`).  The mover lane does all the rest in one
// polling loop that blocks only on its own bulk groups:
//   - a handed-back tile: issue its store and keep going; up to NSLOT stores may be reading shared memory at once;
//   - a free slot: take the next tile from the work order and issue its load (or, for a tile with a dependency, poll it
//     until it is met, so that a waiting tile holds up neither the stores nor the publications);
//   - nothing else to do: publish a pending tile (W::PUBLISH) once every store is complete, or else wait for the oldest
//     store to have READ its slot (cp.async.bulk.wait_group.read) and free that slot -- slots are freed in ring order.
// After the last tile, the mover puts NGROUP end markers (descriptor role -1, no bytes) into the next positions, one for
// each group, and leaves when every store is complete.
// Proxy order of the hand-over: consumers' smem writes, fence.proxy.async.shared::cta, group barrier, `done` arrive; the
// mover's mbarrier test_wait, then its TMA store.
//
// W, the work order: next(n, d) fills the descriptor d[4] = {role, x, y, id} of position n and returns TMA_W_END,
// TMA_W_LOAD or TMA_W_WAIT; dep_met(d), load(n, d, buf, bar), store(n, d, buf) (no commit), publish(d) for a role-0 tile
// whose store is complete (W::PUBLISH), transform(d, buf, lut, bid, lt) and finish() (mover, after the last store).
enum { TMA_W_END = 0, TMA_W_LOAD = 1, TMA_W_WAIT = 2 };

template <class S, typename T, int C, int PROBE, class W>
__device__ __forceinline__ void tma_ring(W& w, const cx<T>* lut, unsigned long long* stamps)
{
    using G_ = TmaGeom<S, T, C>;
    constexpr int NT = G_::NT, NSLOT = G_::NSLOT, NGROUP = G_::NGROUP;
    constexpr bool STAMPS = (PROBE & TMA_STAMPS) != 0;
    static_assert(TMA_CONSUMERS % NT == 0, "the consumers split into whole groups");
    static_assert(NSLOT >= NGROUP + 1, "the ring needs a slot per group and one more");
    extern __shared__ __align__(128) unsigned char tma_raw[];
    cx<T>* const lut_s = reinterpret_cast<cx<T>*>(tma_raw + (size_t)NSLOT * G_::TILE_BYTES);
    uint64_t* const full = reinterpret_cast<uint64_t*>(tma_raw + (size_t)NSLOT * G_::TILE_BYTES + G_::LUT_BYTES);
    uint64_t* const done = full + NSLOT;                            // per slot: the consumers have written the tile back
    int* const desc = reinterpret_cast<int*>(done + NSLOT);         // per slot: role (-1 end), x, y, stamp id
    auto slot = [&](int i) { return reinterpret_cast<cx<T>*>(tma_raw + (size_t)i * G_::TILE_BYTES); };
    auto stamp = [&](int id, int f) {
        if constexpr (STAMPS) stamps[(size_t)(unsigned)id * TMA_NSTAMP + f] = gtime_ns();
    };
    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int i = 0; i < NSLOT; i++) { mbar_init(full + i, 1); mbar_init(done + i, 1); }
        fence_barrier_init();
    }
    for (int i = tid; i < S::lut_size(); i += TMA_CONSUMERS + 32) lut_s[i] = lut[i];
    __syncthreads();

    if (tid >= TMA_CONSUMERS) {
        if (tid != TMA_CONSUMERS) return;
        unsigned n_load = 0;    // next ring position to fill
        unsigned n_store = 0;   // next position the consumers hand back
        unsigned n_free = 0;    // every position below is free: its store has read the slot
        unsigned n_end = 0;     // position of the first end marker, once the work order has ended
        bool ended = false;
        bool waiting = false;   // the tile at n_load waits for its dependency
        bool pend = false;      // the newest role-0 store of a publishing work order is not yet known complete
        int pend_d[4] = {0, 0, 0, 0};
        auto free_upto = [&](unsigned n) {   // positions below n have been read by their stores
            for (; n_free < n; n_free++) {
                if constexpr (STAMPS) {
                    const int* d = desc + (n_free % NSLOT) * 4;
                    stamp(d[3], TMS_FREED);
                    if (!(W::PUBLISH && d[0] == 0)) stamp(d[3], TMS_RETIRED);
                }
            }
        };
        auto publish = [&]() {   // every store issued so far is complete
            stamp(pend_d[3], TMS_RETIRED);
            w.publish(pend_d);
            pend = false;
        };
        SpinGuard guard;
        for (;;) {
            bool acted = false;
            // a transformed tile: store it
            const int ss = (int)(n_store % NSLOT);
            if (n_store < n_load && (!ended || n_store < n_end) && mbar_test_wait(done + ss, (n_store / NSLOT) & 1)) {
                const int* d = desc + ss * 4;
                w.store(n_store, d, slot(ss));
                tma_commit();
                stamp(d[3], TMS_STORE);
                if (pend) {   // the pending tile's store is older than this one
                    tma_wait_all<1>();
                    free_upto(n_store);
                    publish();
                }
                if (W::PUBLISH && d[0] == 0) { pend = true; pend_d[1] = d[1]; pend_d[3] = d[3]; }
                n_store++;
                acted = true;
            }
            // a free slot: the next tile's load, or an end marker for the next group
            if (!waiting && n_load < n_free + NSLOT && (!ended || n_load < n_end + NGROUP)) {
                const int s = (int)(n_load % NSLOT);
                int* d = desc + s * 4;
                if (ended) {
                    d[0] = -1;
                    tma_mbar_arrive(full + s);
                    n_load++;
                } else {
                    const int r = w.next(n_load, d);
                    if (r == TMA_W_END) {
                        n_end = n_load;
                        ended = true;
                        continue;   // the marker goes in on the next round
                    }
                    if constexpr (STAMPS) {
                        stamps[(size_t)(unsigned)d[3] * TMA_NSTAMP + TMS_WHO] = blockIdx.x * 2u + (d[0] == 1 && W::PUBLISH ? 1u : 0u);
                        stamp(d[3], TMS_TICKET);
                    }
                    if (r == TMA_W_LOAD) {
                        stamp(d[3], TMS_DEP);
                        mbar_expect_tx(full + s, G_::TILE_BYTES);
                        w.load(n_load, d, slot(s), full + s);
                        stamp(d[3], TMS_LOAD);
                        n_load++;
                    } else waiting = true;
                }
                acted = true;
            }
            if (waiting) {
                const int s = (int)(n_load % NSLOT);
                const int* d = desc + s * 4;
                if (w.dep_met(d)) {
                    stamp(d[3], TMS_DEP);
                    mbar_expect_tx(full + s, G_::TILE_BYTES);
                    w.load(n_load, d, slot(s), full + s);
                    stamp(d[3], TMS_LOAD);
                    waiting = false;
                    n_load++;
                    acted = true;
                }
            }
            if (acted) { guard = SpinGuard{}; continue; }
            if (ended && n_load == n_end + NGROUP && n_store == n_end) break;
            // nothing to do: publish the pending tile now rather than with the next store, since tiles of other CTAs (or
            // the very tile this CTA waits on) may be waiting for it; otherwise free the oldest slot whose store has read it
            if (pend) {
                tma_wait_all<0>();
                free_upto(n_store);
                publish();
            } else if (n_free < n_store) {
                tma_wait_read_dyn<NSLOT>((int)(n_store - n_free - 1));
                free_upto(n_free + 1);
            } else {
                if (waiting) __nanosleep(64);
                guard.tick();
            }
        }
        tma_wait_all<0>();
        free_upto(n_store);
        if (pend) publish();
        w.finish();
        return;
    }

    // ---- consumers: group g transforms positions g, g + NGROUP, ... and hands each back to the mover ----
    const int g = tid / NT, lt = tid % NT, bid = 1 + g;
    for (unsigned n = g;; n += NGROUP) {
        const int s = (int)(n % NSLOT);
        unsigned long long ready = 0;
        if constexpr (STAMPS) ready = gtime_ns();
        mbar_wait(full + s, (n / NSLOT) & 1);
        const int* d = desc + s * 4;
        if (d[0] < 0) break;   // end marker: this group's last position
        if constexpr (STAMPS) {
            if (lt == 0) {
                stamps[(size_t)(unsigned)d[3] * TMA_NSTAMP + TMS_READY] = ready;
                stamp(d[3], TMS_FULL);
            }
        }
        if constexpr ((PROBE & TMA_MOVE) == 0) w.transform(d, slot(s), lut_s, bid, lt);   // the twin: the slot leaves as it arrived
        tma_fence_smem_writes();   // generic-proxy writes -> visible to the mover's TMA store
        tma_sync<NT>(bid);
        if (lt == 0) {
            stamp(d[3], TMS_DONE);
            tma_mbar_arrive(done + s);
        }
    }
}

// ---- per-axis passes ------------------------------------------------------------------------------------------------------
// NT = S::T * C threads and a TMA_PASS_NSLOT-slot ring; thread 0 issues every load and store: the load of tile i + 2 goes
// into the slot whose store (tile i - 1) has been read.  A mover lane (tma_ring) measured slower for TMA_XF at 512^3 fp64
// on H100: 1.64 against 1.57 ms (DESIGN.md 3.4), so the passes keep this structure.
template <class S, typename T, int C, int MODE>
__global__ void __launch_bounds__(S::T* C, 1) fft_tma_pass_kernel(const TmaArgs<T> A, const __grid_constant__ CUtensorMap map_in, const __grid_constant__ CUtensorMap map_out)
{
    using G_ = TmaGeom<S, T, C>;
    constexpr int N = S::N, NT = G_::NT, ROWS = G_::ROWS, NBOX = G_::NBOX, NSLOT = TMA_PASS_NSLOT;
    constexpr bool IN_LINES = MODE == TMA_Z || MODE == TMA_XB, OUT_LINES = MODE == TMA_Z || MODE == TMA_XF;
    extern __shared__ __align__(128) unsigned char tma_raw[];
    cx<T>* const lut_s = reinterpret_cast<cx<T>*>(tma_raw + (size_t)NSLOT * G_::TILE_BYTES);
    uint64_t* const full = reinterpret_cast<uint64_t*>(tma_raw + (size_t)NSLOT * G_::TILE_BYTES + G_::LUT_BYTES);
    auto slot = [&](int i) { return reinterpret_cast<cx<T>*>(tma_raw + (size_t)i * G_::TILE_BYTES); };
    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int i = 0; i < NSLOT; i++) mbar_init(full + i, 1);
        fence_barrier_init();
    }
    for (int i = tid; i < S::lut_size(); i += NT) lut_s[i] = A.lut[i];
    __syncthreads();
    const long long mine = A.ntiles > blockIdx.x ? (A.ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    auto load = [&](long long i) {   // thread 0
        const int s = (int)(i % NSLOT);
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
        for (long long i = 0; i < mine && i < NSLOT - 1; i++) load(i);
    for (long long i = 0; i < mine; i++) {
        const int s = (int)(i % NSLOT);
        cx<T>* buf = slot(s);
        mbar_wait(full + s, (uint32_t)((i / NSLOT) & 1));
        tma_transform<S, T, MODE, C, NT>(buf, lut_s, 1, tid, A.inv != 0, A.do_scale != 0, A.scale);
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
            if (i + NSLOT - 1 < mine) {
                tma_wait_read<1>();     // the store of tile i-1 has drained its slot, which tile i+2 reuses
                load(i + NSLOT - 1);
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
// It runs on tma_ring: the mover draws a ticket for each free slot, loads a Y tile only after its plane's counter has reached
// the target (polled), and publishes a Z tile (plane counter += 1) once its store is complete -- as soon as the mover has
// nothing else to do (wait_group 0), or when a later store has been issued and everything older is complete (wait_group 1).
// Why a mover (csrc/tools/t0_profile.py, DESIGN.md 3.4): when consumer thread 0 issued the stores, it waited for the
// previous store's completion before every tile, and each slot stayed held until its store was complete.
// Deadlock freedom, whatever the residency: a Y ticket waits only for Z tickets of its plane, and all of them are lower.
// Each of those was drawn by a running mover with a free slot, so its load is in flight; the tiles ahead of it in that CTA's
// ring have still lower tickets (tickets rise per CTA), so by induction they land, and the consumer groups, who wait for
// nothing but landed slots in their own positions, hand them back.  (Every group does: a group's positions are taken in ring
// order, and the ring holds only loaded tiles ahead of the waiting one.)  The Z tile's store is then issued, and it is
// published without waiting for a later tile to land: the mover publishes it the first time it finds nothing else to do,
// which it must while the next ticket is a Y tile still waiting for its plane, and at the latest with the next store.
// Proxy order: Z tile: store's wait_group, fence.proxy.async, __threadfence, counter add; Y tile: ld.acquire.gpu of the
// counter, fence.proxy.async, tensor load.
// L2 policy per instruction (createpolicy): the slab is read once and the finished Y columns are not read again by this
// kernel, so the Z loads and the Y stores are evict_first; the Z stores of the intermediate are evict_last, so that they
// survive until their Y tiles read them.  At 512^3 fp64 on H100 the three hints together take t0 from 2.90 to 2.30 ms at
// lag 4 (DESIGN.md 3.4).  No persisting-L2 carve-out is used: that is a device-wide setting.
template <typename T> struct TmaFusedArgs {
    const cx<T>* src;    // Z role input (dense planes of N x N)
    cx<T>* mid;          // Z role output, Y role input and output (described by map_mid)
    const cx<T>* lut;
    unsigned long long* stamps;   // TMA_STAMPS instantiations only: TMA_NSTAMP words per ticket; null in the library
};

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

// descriptor: {role 0 = Z / 1 = Y, plane, tile index in the plane's role, ticket}
template <class S, typename T, int C> struct TmaFusedWork {
    using G_ = TmaGeom<S, T, C>;
    static constexpr bool PUBLISH = true;
    const TmaFusedArgs<T>& A;
    const FusedCtl& F;
    const CUtensorMap* map_mid;
    Fused2Order o;
    __device__ int next(unsigned, int* d) const
    {
        const unsigned t = atomicAdd(F.ticket, 1u);
        if (t >= o.total) return TMA_W_END;
        bool z;
        unsigned plane, idx;
        fused2_decode(o, t, z, plane, idx);
        d[0] = z ? 0 : 1; d[1] = (int)plane; d[2] = (int)idx; d[3] = (int)t;
        return z ? TMA_W_LOAD : TMA_W_WAIT;
    }
    __device__ bool dep_met(const int* d) const   // every Z tile of the plane is stored
    {
        unsigned long long v;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(F.plane_done + d[1]) : "memory");
        if (v < F.target) return false;
        asm volatile("fence.proxy.async;" ::: "memory");   // the acquired data is read through the async proxy
        return true;
    }
    // policies made at the point of use: held across the mover's loop they cost spill slots
    __device__ void load(unsigned, const int* d, cx<T>* buf, uint64_t* bar) const
    {
        if (d[0] == 0) tma_bulk_g2s_hint(buf, A.src + ((long long)d[1] * o.GA + d[2]) * (C * S::N), G_::TILE_BYTES, bar, l2_policy_evict_first());
        else {
#pragma unroll
            for (int r = 0; r < G_::NBOX; r++) tma_tensor_g2s_3d(buf + r * G_::ROWS * C, map_mid, d[2] * C * 2, r * G_::ROWS, d[1], bar);
        }
    }
    __device__ void store(unsigned, const int* d, const cx<T>* buf) const
    {
        if (d[0] == 0) tma_bulk_s2g_hint(A.mid + ((long long)d[1] * o.GA + d[2]) * (C * S::N), buf, G_::TILE_BYTES, l2_policy_evict_last());
        else {
            const uint64_t write_once = l2_policy_evict_first();
#pragma unroll
            for (int r = 0; r < G_::NBOX; r++) tma_tensor_s2g_3d_hint(map_mid, d[2] * C * 2, r * G_::ROWS, d[1], buf + r * G_::ROWS * C, write_once);
        }
    }
    __device__ void publish(const int* d) const   // the Z tile's store is complete
    {
        asm volatile("fence.proxy.async;" ::: "memory");
        __threadfence();
        atomicAdd(F.plane_done + d[1], 1ull);
    }
    __device__ void transform(const int* d, cx<T>* buf, const cx<T>* lut, int bid, int lt) const
    {
        if (d[0] == 0) tma_transform<S, T, TMA_Z, C, G_::NT>(buf, lut, bid, lt, false, false, T(1));
        else tma_transform<S, T, TMA_Y, C, G_::NT>(buf, lut, bid, lt, false, false, T(1));
    }
    __device__ void finish() const   // the last CTA to leave re-arms the ticket counter
    {
        const unsigned left = atomicAdd(F.ticket + 1, 1u);
        if (left == gridDim.x - 1) { F.ticket[0] = 0; F.ticket[1] = 0; __threadfence(); }
    }
};

template <class S, typename T, int C, int PROBE>
__device__ __forceinline__ void tma_fused_zy_body(const TmaFusedArgs<T>& A, const FusedCtl& F, const CUtensorMap* map_mid)
{
    TmaFusedWork<S, T, C> w{A, F, map_mid, fused2_prepare(F)};
    tma_ring<S, T, C, PROBE>(w, A.lut, A.stamps);
}

template <class S, typename T, int C>
__global__ void __launch_bounds__(TMA_CONSUMERS + 32, 1) fft_tma_fused_zy_kernel(const TmaFusedArgs<T> A, const FusedCtl F,
                                                                                 const __grid_constant__ CUtensorMap map_mid)
{
    tma_fused_zy_body<S, T, C, 0>(A, F, &map_mid);
}

// the measurement instantiations (TMA_MOVE, TMA_STAMPS), launched like fft_tma_fused_zy_kernel
template <class S, typename T, int C, int PROBE>
__global__ void __launch_bounds__(TMA_CONSUMERS + 32, 1) fft_tma_fused_zy_probe_kernel(const TmaFusedArgs<T> A, const FusedCtl F,
                                                                                       const __grid_constant__ CUtensorMap map_mid)
{
    tma_fused_zy_body<S, T, C, PROBE>(A, F, &map_mid);
}

}  // namespace dfft
