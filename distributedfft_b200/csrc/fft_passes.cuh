// fft_passes.cuh -- the one tile kernel all passes instantiate.
//
// A "tile" is C lines of N points.  Addressing is affine with an optional chunk table:
//   element (tile, c, e) lives at  base + a*SA + b*SB + c*cs + e*es,  (a, b) = (tile / G, tile % G)
// which covers
//   Z pass  (t0, contiguous lines)          cs = N2, es = 1          thread map MAP_T
//   Y pass  (t0, stride N2, +fused t1 pack) cs = 1,  es = N2         thread map MAP_C
//   X pass  (t3, fused unpack + transpose)  load cs = 1, es = n1_l*N2 (MAP_C); store cs = N0, es = 1 (MAP_T)
// and their backward twins.  With CHUNK_* the position e is split as q = e / ediv, el = e % ediv
// and the address becomes  cptr[q] + a*SAq[q] + b*SB + c*cs + el*es : that is the reference's
// per-destination pack (kernel_func.cpp:73-86) folded into the Y-pass store, with cptr[q] either
// the local send buffer chunk or -- fused all-to-all -- the peer's receive buffer mapped over
// NVLink (fft_mpi_3d_api.cpp:613-630 hipMemcpyPeerAsync into nodeDataDev[i]).
#pragma once
#include "fft_core.cuh"

namespace dfft {

enum { MAP_T = 0, MAP_C = 1 };
constexpr int DFFT_MAX_CHUNKS = 32;

struct Affine {
    long long SA, SB, cs, es;
};

struct ChunkTab {
    void* cptr[DFFT_MAX_CHUNKS];        // base pointer of chunk q (already includes the fixed offset)
    long long SAq[DFFT_MAX_CHUNKS];     // stride of tile coordinate `a` inside chunk q
    int ediv;                           // chunk extent along the transform axis (yd or xd)
    int nchunks;
};

template <typename T> struct TileArgs {
    const cx<T>* in;
    cx<T>* out;
    const cx<T>* lut;      // per-length twiddle table (Sched::lut_size() entries)
    Affine ia, oa;
    long long ntiles;      // total tiles
    int G;                 // tiles per `a`
    int W;                 // columns per `a` (for the ragged last tile: valid = min(C, W - b*C))
    T scale;               // applied on store when do_scale
    int inv;               // 1: inverse transform (e^{+i..}), unnormalised
    int do_scale;
    ChunkTab ci, co;       // used when CHUNK_IN / CHUNK_OUT
    const void* gen;       // host pointer to the GenSched of a generic-length entry (read by its launcher only)
    long long tw_n;        // four-step epilogue (EPI): multiply output (column col, point k) by e^{-2 pi i col*k / tw_n}; 0 = off
    // completion signal folded into the kernel (stream-pipelined forward): when sig_n > 0 the last CTA to finish publishes
    // sig_val at sig[0..sig_n) -- the per-part arrival flags on the receiving devices, peer-mapped -- with system-scope release
    // semantics after every CTA's (peer) stores; done_ctr counts finished CTAs and is re-armed by that last CTA
    unsigned long long* sig[DFFT_MAX_CHUNKS];
    unsigned long long sig_val;
    unsigned int* done_ctr;
    int sig_n;
    // start gate folded into the kernel: when wait_n > 0 every CTA first polls wait_flags[0..wait_n) (system-scope acquire) until
    // they reach wait_val -- "every sender's data has arrived" / "every receiver has consumed the previous execute"
    const unsigned long long* wait_flags;
    unsigned long long wait_val;
    int wait_n;
    int max_ctas_per_sm;   // launcher only: cap on resident CTAs per SM (0 = occupancy limit); the stream-pipelined forward path
                           // leaves SM slots free so that the send-side Y parts and the receive-side X parts co-reside
};

template <class S, typename T, int C, bool PINGPONG>
struct TileSmem {
    static constexpr int LS = SmemGeom<T>::line(S::N, C);
    static constexpr size_t exch_bytes = ((S::NSTAGES > 1 ? (PINGPONG ? 2 : 1) : 0) * (size_t)C * LS * sizeof(cx<T>) + 15) / 16 * 16;
    static constexpr size_t lut_bytes = (size_t)((S::lut_size() * sizeof(cx<T>) + 15) / 16 * 16);
    static constexpr size_t tab_bytes = (size_t)S::N * sizeof(int2) * 2 + 2 * DFFT_MAX_CHUNKS * 16;
    static constexpr size_t bytes(bool chunked) { return exch_bytes + lut_bytes + 16 + (chunked ? tab_bytes : 0); }
};

// barrier over the threads that share exchange data: the whole CTA, or -- LSYNC, line-major thread map on both sides -- only
// the S::T threads of one line (named barrier 1 + line), which decouples the lines of a tile from each other
template <bool LSYNC, int TT> __device__ __forceinline__ void exch_sync(int line)
{
    if constexpr (LSYNC) asm volatile("bar.sync %0, %1;" ::"r"(line + 1), "n"(TT) : "memory");
    else __syncthreads();
}

template <class S, int s, typename T, int C, int MAPIN, int MAPOUT, bool TWREG, bool PINGPONG, bool LSYNC = false>
struct StageRunner {
    static_assert(!LSYNC || (MAPIN == MAP_T && MAPOUT == MAP_T && S::T % 32 == 0 && C <= 15), "line-level barriers need whole warps per line and at most 15 lines");
    static constexpr int LAST = S::NSTAGES - 1;
    static constexpr int LS = SmemGeom<T>::line(S::N, C);
    // thread (t_in, c_in) for every stage but the last, (t_out, c_out) for the last one
    // `hook` runs once, right after the first stage's butterflies have consumed the loaded registers
    template <class Hook>
    static __device__ __forceinline__ void run(cx<T>* v, int t_in, int c_in, int t_out, int c_out, cx<T>* exch,
                                               int& pp, const cx<T>* lut, const cx<T>* twr, Hook&& hook)
    {
        const int t = (s == LAST) ? t_out : t_in;
        stage_compute<S, s, T, TWREG>(v, t, lut, twr);
        if constexpr (s == 0) hook();
        if constexpr (s < LAST) {
            cx<T>* buf = exch + (PINGPONG ? (size_t)pp * C * LS : 0);
            if constexpr (!PINGPONG) exch_sync<LSYNC, S::T>(c_in);   // previous readers of the single buffer are done
            stage_scatter<S, s, T>(v, t_in, buf + c_in * LS);
            exch_sync<LSYNC, S::T>(c_in);
            if constexpr (s + 1 == LAST) stage_gather<S, T>(v, t_out, buf + c_out * LS);
            else stage_gather<S, T>(v, t_in, buf + c_in * LS);
            pp ^= 1;
            StageRunner<S, s + 1, T, C, MAPIN, MAPOUT, TWREG, PINGPONG, LSYNC>::run(v, t_in, c_in, t_out, c_out, exch, pp, lut,
                                                                           twr + S::tw_regs(s), hook);
        }
    }
};

template <class S, int s, typename T> struct TwLoader {
    static __device__ __forceinline__ void run(cx<T>* twr, int t_in, int t_out, const cx<T>* lut)
    {
        if constexpr (s < S::NSTAGES) {
            if constexpr (s > 0) stage_load_tw<S, s, T>(twr, s == S::NSTAGES - 1 ? t_out : t_in, lut);
            TwLoader<S, s + 1, T>::run(twr + S::tw_regs(s), t_in, t_out, lut);
        }
    }
};

template <int MAP, int C, int TT> __device__ __forceinline__ void thread_map(int tid, int& t, int& c)
{
    if constexpr (MAP == MAP_T) { t = tid % TT; c = tid / TT; }
    else { c = tid % C; t = tid / C; }
}

// streaming accesses: every element is touched exactly once per pass, so keep it out of L1
template <typename C_> __device__ __forceinline__ C_ ld_stream(const C_* p) { return __ldcg(p); }
template <typename C_> __device__ __forceinline__ void st_stream(C_* p, C_ v) { __stcg(p, v); }

// e^{-2 pi i m/n} evaluated on the fly (four-step twiddle between the two passes of a long 1-D transform)
template <typename T> __device__ __forceinline__ cx<T> unit_root(long long m, long long n)
{
    double sn, cs;
    sincospi(-2.0 * (double)m / (double)n, &sn, &cs);
    return mk<T>((T)cs, (T)sn);
}

// L2 eviction-priority hints (createpolicy + .L2::cache_hint): 1 = evict_first (streamed once), 2 = evict_last (the
// intermediate of the fused kernels, which must survive in L2 until the second role has read it)
template <int H> __device__ __forceinline__ unsigned long long l2_policy()
{
    unsigned long long p = 0;
    if constexpr (H == 1) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    if constexpr (H == 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ double2 ld_hint(const double2* p, unsigned long long pol)
{
    double2 v;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;" : "=d"(v.x), "=d"(v.y) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ float2 ld_hint(const float2* p, unsigned long long pol)
{
    float2 v;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f32 {%0,%1}, [%2], %3;" : "=f"(v.x), "=f"(v.y) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void st_hint(double2* p, double2 v, unsigned long long pol)
{
    asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1,%2}, %3;" ::"l"(p), "d"(v.x), "d"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint(float2* p, float2 v, unsigned long long pol)
{
    asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1,%2}, %3;" ::"l"(p), "f"(v.x), "f"(v.y), "l"(pol) : "memory");
}
template <int H, typename C_> __device__ __forceinline__ C_ ld_pol(const C_* p, unsigned long long pol)
{
    if constexpr (H == 0) return ld_stream(p);
    else return ld_hint(p, pol);
}
template <int H, typename C_> __device__ __forceinline__ void st_pol(C_* p, C_ v, unsigned long long pol)
{
    if constexpr (H == 0) st_stream(p, v);
    else st_hint(p, v, pol);
}

// Called by every thread of a CTA before its first load (see TileArgs::wait_flags).
template <typename T>
__device__ __forceinline__ void wait_flags_at_start(const TileArgs<T>& A)
{
    if (A.wait_n <= 0) return;
    if ((int)threadIdx.x < A.wait_n) {
        unsigned long long v;
        SpinGuard guard;
        for (;;) {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(A.wait_flags + threadIdx.x) : "memory");
            if (v >= A.wait_val) break;
            __nanosleep(100);
            guard.tick();
        }
    }
    __syncthreads();
}

// Called by every thread of a CTA after its last store.  Orders the CTA's (peer) stores at system scope, counts the CTA and --
// in the last CTA of the grid -- publishes the value at the flag addresses.  Receivers poll with ld.acquire.sys.
template <typename T>
__device__ __forceinline__ void signal_when_grid_done(const TileArgs<T>& A)
{
    if (A.sig_n <= 0) return;
    __syncthreads();          // the CTA's stores happen-before thread 0's fence (bar.sync), which is cumulative over them
    if (threadIdx.x == 0) {
        __threadfence_system();
        const unsigned prev = atomicAdd(A.done_ctr, 1u);
        if (prev == gridDim.x - 1) {
            *A.done_ctr = 0;
            __threadfence_system();
            for (int q = 0; q < A.sig_n; q++)
                asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(A.sig[q]), "l"(A.sig_val) : "memory");
        }
    }
}

// per-thread asynchronous global -> shared copies (LDGSTS): the next tile's elements are fetched into the
// thread's private staging slots while the current tile is being transformed
template <int BYTES> __device__ __forceinline__ void cp_async(void* dst_smem, const void* src)
{
    if constexpr (BYTES == 16)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
    else
        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// ------------------------------------------------------------------------------------------
// TileOp: everything one pass does to one tile, as a reusable device-side unit.  `setup` stages the
// twiddle tile (TMA) and the chunk tables into the CTA's shared memory once; `run` loads a tile,
// runs the Stockham stages and stores it.  fft_tile_kernel wraps one TileOp; fft_fused2_kernel
// wraps two (Z then Y, or Y then Z) whose intermediate stays in L2.
// Shared-memory carve-up of one TileOp (offsets from its base):
//   [0, exch_bytes) exchange buffer | lut_bytes twiddles | 16 B mbarrier | tab_bytes chunk tables
// ------------------------------------------------------------------------------------------
template <class S, typename T, int C, int MAPIN, int MAPOUT, bool TWREG, bool CHUNK_IN, bool CHUNK_OUT, bool PINGPONG, bool PF = false,
          int HIN = 0, int HOUT = 0, bool EPI = false, bool LSYNC = false>
struct TileOp {
    using SM = TileSmem<S, T, C, PINGPONG>;
    static constexpr int R = S::R, TT = S::T, NT = S::T * C;
    static constexpr bool CHUNKED = CHUNK_IN || CHUNK_OUT;
    // PF: software prefetch.  Element u of thread tid of the NEXT tile is copied asynchronously into the private slot
    // stage[u * NT + tid] (conflict-free, never touched by another thread, so no barrier is involved).
    static constexpr size_t stage_bytes = PF ? (size_t)R * NT * sizeof(cx<T>) : 0;
    static constexpr size_t aux_bytes = SM::lut_bytes + 16 + (CHUNKED ? SM::tab_bytes : 0) + stage_bytes;   // everything but the exchange buffer
    static constexpr int NTW = TWREG ? (S::tw_regs_total() > 0 ? S::tw_regs_total() : 1) : 1;

    struct Ctx {
        cx<T>* exch;
        cx<T>* lut_s;
        int2 *etab_i, *etab_o;
        char **cptr_i, **cptr_o;
        long long *saq_i, *saq_o;
        int t_in, c_in, t_out, c_out;
        int pp;
        cx<T>* stage;
        unsigned long long pol_in, pol_out;   // L2 cache policies (HIN / HOUT)
    };

    // exch: exchange buffer (SM::exch_bytes, may be shared with another TileOp); aux: aux_bytes of this op's own
    static __device__ __forceinline__ void setup(const TileArgs<T>& A, unsigned char* exch, unsigned char* aux, Ctx& k)
    {
        const int tid = threadIdx.x;
        k.exch = reinterpret_cast<cx<T>*>(exch);
        k.lut_s = reinterpret_cast<cx<T>*>(aux);
        uint64_t* bar = reinterpret_cast<uint64_t*>(aux + SM::lut_bytes);
        unsigned char* tabs = aux + SM::lut_bytes + 16;
        k.etab_i = reinterpret_cast<int2*>(tabs);
        k.etab_o = k.etab_i + S::N;
        k.cptr_i = reinterpret_cast<char**>(k.etab_o + S::N);
        k.cptr_o = k.cptr_i + DFFT_MAX_CHUNKS;
        k.saq_i = reinterpret_cast<long long*>(k.cptr_o + DFFT_MAX_CHUNKS);
        k.saq_o = k.saq_i + DFFT_MAX_CHUNKS;
        k.pp = 0;
        k.pol_in = l2_policy<HIN>();
        k.pol_out = l2_policy<HOUT>();
        k.stage = reinterpret_cast<cx<T>*>(aux + SM::lut_bytes + 16 + (CHUNKED ? SM::tab_bytes : 0));
        thread_map<MAPIN, C, TT>(tid, k.t_in, k.c_in);
        thread_map<MAPOUT, C, TT>(tid, k.t_out, k.c_out);
        // twiddle tile: global -> shared by one TMA bulk copy
        stage_twiddles_tma<T>(k.lut_s, A.lut, S::lut_size(), bar);
        if constexpr (CHUNKED) {
            for (int e = tid; e < S::N; e += NT) {
                if (CHUNK_IN) { int q = e / A.ci.ediv; q = q < A.ci.nchunks ? q : A.ci.nchunks - 1; k.etab_i[e] = make_int2(q, e - q * A.ci.ediv); }
                if (CHUNK_OUT) { int q = e / A.co.ediv; q = q < A.co.nchunks ? q : A.co.nchunks - 1; k.etab_o[e] = make_int2(q, e - q * A.co.ediv); }
            }
            if (tid < DFFT_MAX_CHUNKS) {
                if (CHUNK_IN) { k.cptr_i[tid] = (char*)A.ci.cptr[tid]; k.saq_i[tid] = A.ci.SAq[tid]; }
                if (CHUNK_OUT) { k.cptr_o[tid] = (char*)A.co.cptr[tid]; k.saq_o[tid] = A.co.SAq[tid]; }
            }
            __syncthreads();
        }
    }

    static __device__ __forceinline__ void load_twiddles(const Ctx& k, cx<T>* twr)
    {
        if constexpr (TWREG) TwLoader<S, 0, T>::run(twr, k.t_in, k.t_out, k.lut_s);
    }

    // issue the asynchronous loads of `tile` into this thread's staging slots (PF only)
    static __device__ __forceinline__ void prefetch(const TileArgs<T>& A, const Ctx& k, long long tile)
    {
        if constexpr (PF) {
            const int t_in = k.t_in, c_in = k.c_in;
            const long long a = tile / A.G;
            const int b = (int)(tile - a * A.G);
            const bool ok = b * C + c_in < A.W;
            cx<T>* slot = k.stage + threadIdx.x;
            if constexpr (!CHUNK_IN) {
                const cx<T>* p = A.in + a * A.ia.SA + b * A.ia.SB + c_in * A.ia.cs + (long long)t_in * A.ia.es;
#pragma unroll
                for (int u = 0; u < R; u++) {
                    if (ok) cp_async<sizeof(cx<T>)>(slot + u * NT, p + (long long)u * TT * A.ia.es);
                    else slot[u * NT] = mk<T>(0, 0);
                }
            } else {
                const long long off = b * A.ia.SB + c_in * A.ia.cs;
#pragma unroll
                for (int u = 0; u < R; u++) {
                    const int2 qe = k.etab_i[t_in + u * TT];
                    const cx<T>* p = reinterpret_cast<const cx<T>*>(k.cptr_i[qe.x]) + a * k.saq_i[qe.x] + off + (long long)qe.y * A.ia.es;
                    if (ok) cp_async<sizeof(cx<T>)>(slot + u * NT, p);
                    else slot[u * NT] = mk<T>(0, 0);
                }
            }
            cp_async_commit();
        }
    }

    // next_tile < 0: nothing to prefetch.  With PF the caller must have prefetched `tile` before the first call.
    static __device__ __forceinline__ void run(const TileArgs<T>& A, Ctx& k, long long tile, const cx<T>* twr, long long next_tile = -1)
    {
        const bool inv = A.inv != 0;   // inverse transform = swap(re,im) -> forward -> swap(re,im)
        const bool do_scale = A.do_scale != 0;
        const int t_in = k.t_in, c_in = k.c_in, t_out = k.t_out, c_out = k.c_out;
        const long long a = tile / A.G;
        const int b = (int)(tile - a * A.G);
        cx<T> v[R];
        if constexpr (PF) {
            cp_async_wait_all();
            const cx<T>* slot = k.stage + threadIdx.x;
#pragma unroll
            for (int u = 0; u < R; u++) v[u] = slot[u * NT];
            if (inv) {
#pragma unroll
                for (int u = 0; u < R; u++) v[u] = cswap(v[u]);
            }
        } else {
            const bool ok = b * C + c_in < A.W;
            if constexpr (!CHUNK_IN) {
                const cx<T>* p = A.in + a * A.ia.SA + b * A.ia.SB + c_in * A.ia.cs + (long long)t_in * A.ia.es;
#pragma unroll
                for (int u = 0; u < R; u++) v[u] = ok ? ld_pol<HIN>(p + (long long)u * TT * A.ia.es, k.pol_in) : mk<T>(0, 0);
            } else {
                const long long off = b * A.ia.SB + c_in * A.ia.cs;
#pragma unroll
                for (int u = 0; u < R; u++) {
                    const int2 qe = k.etab_i[t_in + u * TT];
                    const cx<T>* p = reinterpret_cast<const cx<T>*>(k.cptr_i[qe.x]) + a * k.saq_i[qe.x] + off + (long long)qe.y * A.ia.es;
                    v[u] = ok ? ld_pol<HIN>(p, k.pol_in) : mk<T>(0, 0);
                }
            }
            if (inv) {
#pragma unroll
                for (int u = 0; u < R; u++) v[u] = cswap(v[u]);
            }
        }
        // the staging slots are free once the first stage has consumed the registers loaded from them
        auto hook = [&]() { if constexpr (PF) { if (next_tile >= 0) prefetch(A, k, next_tile); } };
        StageRunner<S, 0, T, C, MAPIN, MAPOUT, TWREG, PINGPONG, LSYNC>::run(v, t_in, c_in, t_out, c_out, k.exch, k.pp, k.lut_s, twr, hook);
        if constexpr (EPI) {   // four-step twiddle W_n^(col * k), applied in the forward domain (before the inverse's swap-back)
            const long long col = (long long)b * C + c_out;
#pragma unroll
            for (int u = 0; u < R; u++) v[u] = cmul(v[u], unit_root<T>((col * (long long)(t_out + u * TT)) % A.tw_n, A.tw_n));
        }
        {
            if (inv) {
#pragma unroll
                for (int u = 0; u < R; u++) v[u] = cswap(v[u]);
            }
            if (do_scale) {
#pragma unroll
                for (int u = 0; u < R; u++) { v[u].x *= A.scale; v[u].y *= A.scale; }
            }
            const bool ok = b * C + c_out < A.W;
            if (ok) {
                if constexpr (!CHUNK_OUT) {
                    cx<T>* p = A.out + a * A.oa.SA + b * A.oa.SB + c_out * A.oa.cs + (long long)t_out * A.oa.es;
#pragma unroll
                    for (int u = 0; u < R; u++) st_pol<HOUT>(p + (long long)u * TT * A.oa.es, v[u], k.pol_out);
                } else {
                    const long long off = b * A.oa.SB + c_out * A.oa.cs;
#pragma unroll
                    for (int u = 0; u < R; u++) {
                        const int2 qe = k.etab_o[t_out + u * TT];
                        cx<T>* p = reinterpret_cast<cx<T>*>(k.cptr_o[qe.x]) + a * k.saq_o[qe.x] + off + (long long)qe.y * A.oa.es;
                        st_pol<HOUT>(p, v[u], k.pol_out);
                    }
                }
            }
        }
    }
};

template <class S, typename T, int C, int MAPIN, int MAPOUT, bool TWREG, bool CHUNK_IN, bool CHUNK_OUT, int MINB,
          bool PINGPONG, bool PF = false, bool EPI = false>
__global__ void __launch_bounds__(S::T* C, MINB) fft_tile_kernel(const TileArgs<T> A)
{
    static_assert(S::valid(), "bad schedule");
    static_assert(S::NSTAGES > 1 || MAPIN == MAPOUT, "a thread-map change needs an exchange");
    using Op = TileOp<S, T, C, MAPIN, MAPOUT, TWREG, CHUNK_IN, CHUNK_OUT, PINGPONG, PF, 0, 0, EPI>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename Op::Ctx k;
    Op::setup(A, smem_raw, smem_raw + Op::SM::exch_bytes, k);
    cx<T> twr[Op::NTW];
    Op::load_twiddles(k, twr);
    wait_flags_at_start<T>(A);
    if (PF && (long long)blockIdx.x < A.ntiles) Op::prefetch(A, k, blockIdx.x);
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        const long long next = tile + gridDim.x;
        Op::run(A, k, tile, twr, next < A.ntiles ? next : -1);
    }
    signal_when_grid_done<T>(A);
}

// ------------------------------------------------------------------------------------------
// Two dependent passes over the same planes in ONE persistent kernel (t0 = Z then Y forward, Y then Z
// backward): the reference runs them as two launches per plane (fft_mpi_3d_api.cpp:496-502), we ran
// them as two full HBM sweeps; here a plane's intermediate is produced and consumed while it is still
// resident in L2 (50 MB on H100), so t0 costs one HBM read + one HBM write of the slab.
//
// Work is handed out by a global ticket counter in an order that interleaves "role A on plane
// x + lag" with "role B on plane x".  A role-B tile waits on its plane's completion counter
// (release/acquire at gpu scope); every lower ticket is held by a running CTA and role-A tiles never
// wait, so the scheme cannot deadlock whatever the residency.  The counters are monotonic
// (target = epoch * tiles-per-plane); the last CTA to leave re-arms the ticket counter.
// ------------------------------------------------------------------------------------------
struct FusedCtl {
    unsigned long long* plane_done;   // [planes]
    unsigned int* ticket;             // [0] next ticket, [1] CTAs that have left
    unsigned long long target;        // plane_done value that means "role A finished this plane in this execute"
    long long planes;
    int GA, GB;                       // tiles per plane of role A / role B
    int lag;                          // role A runs this many planes ahead of role B
};

template <class OpA, class OpB, typename T, int MINB>
__global__ void __launch_bounds__(OpA::NT, MINB) fft_fused2_kernel(const TileArgs<T> A, const TileArgs<T> B, const FusedCtl F)
{
    static_assert(OpA::NT == OpB::NT, "both roles use the whole CTA");
    constexpr size_t exch = OpA::SM::exch_bytes > OpB::SM::exch_bytes ? OpA::SM::exch_bytes : OpB::SM::exch_bytes;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ long long s_ticket;
    typename OpA::Ctx ka;
    typename OpB::Ctx kb;
    OpA::setup(A, smem_raw, smem_raw + exch, ka);
    OpB::setup(B, smem_raw, smem_raw + exch + OpA::aux_bytes, kb);
    cx<T> twa[OpA::NTW], twb[OpB::NTW];
    OpA::load_twiddles(ka, twa);
    OpB::load_twiddles(kb, twb);
    wait_flags_at_start<T>(B);   // the second role's stores may target buffers a peer is still reading (previous execute)

    // ticket arithmetic in 32 bits (a ticket is decoded for every tile; 64-bit divisions cost several hundred cycles each)
    const unsigned GA = (unsigned)F.GA, GB = (unsigned)F.GB, per = GA + GB;
    const unsigned lag = (unsigned)(F.lag < F.planes ? F.lag : F.planes);
    const unsigned headT = lag * GA;                                   // role A on planes [0, lag)
    const unsigned midT = ((unsigned)F.planes - lag) * per;           // pairs: A on plane lag+i, then B on plane i
    const unsigned total = headT + midT + lag * GB;                    // tail: B on the last `lag` planes
    for (;;) {
        __syncthreads();   // previous tile's smem traffic and s_ticket readers are done
        if (threadIdx.x == 0) s_ticket = (long long)atomicAdd(F.ticket, 1u);
        __syncthreads();
        const unsigned t = (unsigned)s_ticket;
        if (t >= total) break;
        bool roleA;
        unsigned plane, idx;
        if (t < headT) { roleA = true; plane = t / GA; idx = t - plane * GA; }
        else if (t < headT + midT) {
            const unsigned u = t - headT, i = u / per, r = u - i * per;
            if (r < GA) { roleA = true; plane = lag + i; idx = r; }
            else { roleA = false; plane = i; idx = r - GA; }
        } else {
            const unsigned u = t - headT - midT, i = u / GB;
            roleA = false; plane = (unsigned)F.planes - lag + i; idx = u - i * GB;
        }
        if (roleA) {
            OpA::run(A, ka, (long long)plane * F.GA + idx, twa);
            __syncthreads();                       // every thread's stores are issued ...
            if (threadIdx.x == 0) {
                __threadfence();                   // ... and ordered before the release
                atomicAdd(F.plane_done + plane, 1ull);
            }
        } else {
            if (threadIdx.x == 0) {
                unsigned long long v;
                SpinGuard guard;
                for (;;) {
                    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(F.plane_done + plane) : "memory");
                    if (v >= F.target) break;
                    __nanosleep(64);
                    guard.tick();   // a lost dependency traps (after DFFT_SPIN_TIMEOUT_NS) instead of hanging the GPU
                }
            }
            __syncthreads();
            OpB::run(B, kb, (long long)plane * F.GB + idx, twb);
        }
    }
    if (B.sig_n > 0) __syncthreads();   // this CTA's (peer) stores happen-before thread 0's cumulative system-scope fence
    if (threadIdx.x == 0) {
        if (B.sig_n > 0) __threadfence_system();
        const unsigned left = atomicAdd(F.ticket + 1, 1u);
        if (left == gridDim.x - 1) {
            F.ticket[0] = 0; F.ticket[1] = 0; __threadfence();
            if (B.sig_n > 0) {   // last CTA: every Y tile of the part is stored -> publish the arrival flags
                __threadfence_system();
                for (int q = 0; q < B.sig_n; q++)
                    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(B.sig[q]), "l"(B.sig_val) : "memory");
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// Send side and receive side of the exchange in ONE persistent kernel (forward, P2P): role A = the Y pass of z-part k
// (its chunked stores land in the peers' receive buffers over NVLink), role B = the X pass of z-part k-1, which has
// already arrived (a one-CTA gate kernel in front of this launch has seen the flags).
// Two separate kernels cannot overlap here -- each wants both CTA slots of every SM, so they serialise or halve each other
// (measured) -- and handing out A and B tiles from ONE ordered ticket stream does not overlap either: a CTA stalled on
// back-pressured NVLink stores keeps its slot, the short B tiles finish, their CTAs draw the next ticket, and soon every slot
// holds a stalled A tile (measured: the B work simply added to the send time).  So the roles are PINNED: the first half of the
// grid (one CTA per SM) prefers A tiles, the second half prefers B tiles, each with its own ticket counter; a CTA only
// crosses over when its own kind is exhausted.  Every SM then always has one slot feeding NVLink and one slot doing the
// HBM-bound X work.  Nothing in this kernel waits on another CTA or another device, so any residency is deadlock free.
// The last CTA to leave publishes the arrival flags of part k (A.sig) after every CTA's stores.
// ------------------------------------------------------------------------------------------
struct YxCtl {
    unsigned int* ticket;                   // [0] next A tile, [1] CTAs that have left, [2] next B tile
    unsigned TA, TB;                        // tiles of role A / role B
};

template <class OpA, class OpB, typename T, int MINB>
__global__ void __launch_bounds__(OpA::NT, MINB) fft_fused_yx_kernel(const TileArgs<T> A, const TileArgs<T> B, const YxCtl F)
{
    static_assert(OpA::NT == OpB::NT, "both roles use the whole CTA");
    constexpr size_t exch = OpA::SM::exch_bytes > OpB::SM::exch_bytes ? OpA::SM::exch_bytes : OpB::SM::exch_bytes;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ int s_role;
    __shared__ unsigned s_idx;
    typename OpA::Ctx ka;
    typename OpB::Ctx kb;
    OpA::setup(A, smem_raw, smem_raw + exch, ka);
    OpB::setup(B, smem_raw, smem_raw + exch + OpA::aux_bytes, kb);
    cx<T> twa[OpA::NTW], twb[OpB::NTW];
    OpA::load_twiddles(ka, twa);
    OpB::load_twiddles(kb, twb);
    const bool prefer_b = blockIdx.x >= (gridDim.x + 1) / 2;
    bool a_left = F.TA > 0, b_left = F.TB > 0;   // thread 0's view: tiles of that kind may still be unclaimed
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) {
            int role = -1;
            unsigned idx = 0;
#pragma unroll
            for (int attempt = 0; attempt < 2; attempt++) {
                const bool try_b = (attempt == 0) == prefer_b;
                if (role < 0 && (try_b ? b_left : a_left)) {
                    const unsigned t = atomicAdd(F.ticket + (try_b ? 2 : 0), 1u);
                    if (t < (try_b ? F.TB : F.TA)) { role = try_b ? 1 : 0; idx = t; }
                    else if (try_b) b_left = false;
                    else a_left = false;
                }
            }
            s_role = role; s_idx = idx;
        }
        __syncthreads();
        const int role = s_role;
        if (role < 0) break;
        if (role == 0) OpA::run(A, ka, (long long)s_idx, twa);
        else OpB::run(B, kb, (long long)s_idx, twb);
    }
    if (A.sig_n > 0) __syncthreads();   // this CTA's peer stores happen-before thread 0's cumulative system-scope fence
    if (threadIdx.x == 0) {
        if (A.sig_n > 0) __threadfence_system();
        const unsigned left = atomicAdd(F.ticket + 1, 1u);
        if (left == gridDim.x - 1) {
            F.ticket[0] = 0; F.ticket[1] = 0; F.ticket[2] = 0; __threadfence();
            if (A.sig_n > 0) {
                __threadfence_system();
                for (int q = 0; q < A.sig_n; q++)
                    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(A.sig[q]), "l"(A.sig_val) : "memory");
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// Forward t0 + t1 + t2 + t3 of one device in ONE persistent kernel (P2P exchange, square planes):
// role A = Z tiles, role B = Y tiles whose chunked store lands in the peers' receive buffers over NVLink,
// role C = X tiles reading this device's receive buffer.  The z axis is cut into K parts; the Y role sends
// part 0 of every plane first (fused with the Z role through L2 as in fft_fused2_kernel), then parts 1..K-1;
// as soon as part k has arrived from all P senders the X role can transform the (y_l, z in part k) lines, so
// all but the last part of t3 runs while the NVLink-bound sends of later parts are still in flight.
//   sender side : tickets are handed out in increasing order, so a CTA that draws a ticket beyond the Y tiles of part k has
//                 stored its last tile of that part: it "passes" the part ONCE (bar.sync, then one fence.sys + atomicAdd by
//                 thread 0 -- not a fence per tile, which serialises every tile behind an NVLink round trip); the CTA whose pass
//                 completes the count publishes arrive[k][me] = epoch at every peer (st.release.sys)
//   receiver    : an X tile of part k polls arrive[k][0..P) with ld.acquire.sys
// Z and Y tiles never wait on a remote device, X tiles wait only on remote Y progress: no cross-device cycle;
// inside the device the ticket order argument of fft_fused2_kernel applies unchanged.
// ------------------------------------------------------------------------------------------
constexpr int DFFT_MAX_PARTS = 8;

struct Fused3Ctl {
    unsigned long long* plane_done;     // [planes]  Z-role completion per plane (monotonic)
    unsigned int* ticket;               // [0] next ticket, [1] CTAs that have left
    unsigned long long* part_done;      // [K]       CTAs that have passed the part (monotonic: epoch * gridDim.x when complete)
    unsigned long long target;          // plane_done value meaning "Z finished this plane in this execute"
    unsigned long long part_target;     // unused (the kernel derives the target from epoch and its grid size)
    unsigned long long epoch;           // value published in / awaited from the arrive flags
    const unsigned long long* my_arrive;                   // [K][DFFT_MAX_CHUNKS] on this device
    unsigned long long* peer_arrive[DFFT_MAX_CHUNKS];      // the same array on device q (peer mapped)
    long long planes, rows;             // local x planes (n0_l), local y rows after the exchange (n1_l)
    int P, me;
    int GA, GB, GBk, GX, GXk, K;        // tiles per plane (Z, Y), Y tiles per plane and part, X tiles per row (all, per part), parts
    int lag;
    // optional timeline (DFFT_DEBUG_TIMELINE): dbg[0..3] minima (start, first X tile), dbg[4..15] maxima / sums, all in ns of %globaltimer
    unsigned long long* dbg;
};

// Ticket order of fft_fused3_kernel (host-callable so that the CPU tests can check it is a bijection onto the tiles
// and respects the dependency order).  All arithmetic is 32-bit with a handful of divisions: a ticket is decoded by every
// CTA for every tile, and the first version's 64-bit proportional interleave cost about a microsecond per ticket.
//   phase 0        : Z on every plane + Y part 0, interleaved like fft_fused2_kernel (Z runs `lag` planes ahead)
//   phase k = 1..K-1: Y part k (LY tiles, plane-major) merged with X part k-1 (LX tiles): first `dly` Y tiles (the part has to
//                    arrive from the peers before its X tiles can run), then blocks of blkA X tiles + blkB Y tiles, then
//                    whatever is left of either kind
//   tail           : X part K-1
// fused3_prepare derives the constants (cheap; once per CTA).
struct Fused3Order {
    unsigned lagp, headT, midT, L0, per0, LY, LX, dly, blkA, blkB, nblk, mixT, phaseT, total;
};
__host__ __device__ inline Fused3Order fused3_prepare(const Fused3Ctl& F)
{
    Fused3Order o{};
    o.lagp = (unsigned)(F.lag < F.planes ? F.lag : F.planes);
    o.per0 = (unsigned)(F.GA + F.GBk);
    o.headT = o.lagp * (unsigned)F.GA;
    o.midT = ((unsigned)F.planes - o.lagp) * o.per0;
    o.L0 = o.headT + o.midT + o.lagp * (unsigned)F.GBk;
    o.LY = (unsigned)F.planes * (unsigned)F.GBk;
    o.LX = (unsigned)F.rows * (unsigned)F.GXk;
    o.dly = o.LY / 4;
    const unsigned ym = o.LY - o.dly;
    // block shape: blkA : blkB ~ LX : ym with blkA + blkB = 8
    unsigned a = ym + o.LX ? (unsigned)((8ull * o.LX + (ym + o.LX) / 2) / (ym + o.LX)) : 4;
    a = a < 1 ? 1 : (a > 7 ? 7 : a);
    o.blkA = a; o.blkB = 8 - a;
    const unsigned nx = o.LX / o.blkA, ny = ym / o.blkB;
    o.nblk = nx < ny ? nx : ny;
    o.mixT = o.nblk * 8u;
    o.phaseT = o.LY + o.LX;
    o.total = o.L0 + (unsigned)(F.K - 1) * o.phaseT + o.LX;
    return o;
}
__host__ __device__ inline long long fused3_total(const Fused3Ctl& F) { return (long long)fused3_prepare(F).total; }
// role 0 = Z, 1 = Y, 2 = X; ypart_floor = lowest Y part whose tiles can still be handed out at tickets >= t
__host__ __device__ inline void fused3_decode(const Fused3Ctl& F, const Fused3Order& o, unsigned t, int& role, int& part, unsigned& plane, unsigned& idx,
                                              int& ypart_floor)
{
    part = 0; plane = 0; idx = 0;
    if (t < o.L0) {
        ypart_floor = 0;
        if (t < o.headT) { role = 0; plane = t / (unsigned)F.GA; idx = t - plane * (unsigned)F.GA; }
        else if (t < o.headT + o.midT) {
            const unsigned u = t - o.headT, i = u / o.per0, r = u - i * o.per0;
            if (r < (unsigned)F.GA) { role = 0; plane = o.lagp + i; idx = r; }
            else { role = 1; plane = i; idx = r - (unsigned)F.GA; }
        } else {
            const unsigned u = t - o.headT - o.midT, i = u / (unsigned)F.GBk;
            role = 1; plane = (unsigned)F.planes - o.lagp + i; idx = u - i * (unsigned)F.GBk;
        }
        return;
    }
    const unsigned u0 = t - o.L0, ph = u0 / o.phaseT, u = u0 - ph * o.phaseT;
    if (ph >= (unsigned)(F.K - 1)) { role = 2; part = F.K - 1; idx = u; ypart_floor = F.K; return; }
    ypart_floor = (int)ph + 1;
    unsigned yi;
    bool isx = false;
    if (u < o.dly) yi = u;
    else {
        const unsigned v = u - o.dly;
        if (v < o.mixT) {
            const unsigned q = v >> 3, r = v & 7u;
            if (r < o.blkA) { isx = true; yi = q * o.blkA + r; }
            else yi = o.dly + q * o.blkB + (r - o.blkA);
        } else {
            const unsigned w = v - o.mixT, remx = o.LX - o.nblk * o.blkA;
            if (w < remx) { isx = true; yi = o.nblk * o.blkA + w; }
            else yi = o.dly + o.nblk * o.blkB + (w - remx);
        }
    }
    if (isx) { role = 2; part = (int)ph; idx = yi; }
    else { role = 1; part = (int)ph + 1; plane = yi / (unsigned)F.GBk; idx = yi - plane * (unsigned)F.GBk; }
}

template <class OpA, class OpB, class OpC, typename T, int MINB>
__global__ void __launch_bounds__(OpA::NT, MINB) fft_fused3_kernel(const TileArgs<T> A, const TileArgs<T> B, const TileArgs<T> Cc, const Fused3Ctl F)
{
    static_assert(OpA::NT == OpB::NT && OpB::NT == OpC::NT, "all roles use the whole CTA");
    constexpr size_t e1 = OpA::SM::exch_bytes > OpB::SM::exch_bytes ? OpA::SM::exch_bytes : OpB::SM::exch_bytes;
    constexpr size_t exch = e1 > OpC::SM::exch_bytes ? e1 : OpC::SM::exch_bytes;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ long long s_ticket;
    typename OpA::Ctx ka;
    typename OpB::Ctx kb;
    typename OpC::Ctx kc;
    OpA::setup(A, smem_raw, smem_raw + exch, ka);
    OpB::setup(B, smem_raw, smem_raw + exch + OpA::aux_bytes, kb);
    OpC::setup(Cc, smem_raw, smem_raw + exch + OpA::aux_bytes + OpB::aux_bytes, kc);
    cx<T> twa[OpA::NTW], twb[OpB::NTW], twc[OpC::NTW];
    OpA::load_twiddles(ka, twa);
    OpB::load_twiddles(kb, twb);
    OpC::load_twiddles(kc, twc);

    const Fused3Order ord = fused3_prepare(F);
    const long long total = (long long)ord.total;
    unsigned long long dbg_t[3] = {0, 0, 0}, dbg_wait = 0, dbg_prev = 0;
    int dbg_n[3] = {0, 0, 0};
    bool dbg_first_x = true, dbg_phase0_done = false;
    if (F.dbg && threadIdx.x == 0) { dbg_prev = gtime_ns(); atomicMin(F.dbg + 0, dbg_prev); }
    int passed = 0;              // Y parts this CTA has passed (uniform over the CTA)
    unsigned arrived_mask = 0;   // parts whose arrival from every sender this CTA has already observed
    // every thread's stores of the previous tile precede the bar.sync at the top of the loop, thread 0's system-scope fence
    // after it is cumulative over them: one fence per CTA and part orders all of the CTA's peer stores of that part
    auto pass_parts = [&](int upto) {
        if (threadIdx.x == 0) {
            for (int k = passed; k < upto; k++) {
                __threadfence_system();
                const unsigned long long old = atomicAdd(F.part_done + k, 1ull);
                if (old + 1 == F.epoch * (unsigned long long)gridDim.x) {   // every CTA of this launch has passed part k
                    __threadfence_system();
                    for (int q = 0; q < F.P; q++)
                        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(F.peer_arrive[q] + (size_t)k * DFFT_MAX_CHUNKS + F.me), "l"(F.epoch) : "memory");
                }
            }
        }
        passed = upto > passed ? upto : passed;
    };
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) s_ticket = (long long)atomicAdd(F.ticket, 1u);
        __syncthreads();
        const long long t = s_ticket;
        int role = 0, part = 0, yfloor = F.K;   // role 0 = Z, 1 = Y, 2 = X
        unsigned plane = 0, idx = 0;            // Z/Y: plane + tile within (plane[, part]); X: idx = tile within the part
        if (t < total) fused3_decode(F, ord, (unsigned)t, role, part, plane, idx, yfloor);
        pass_parts(yfloor);
        if (F.dbg && threadIdx.x == 0 && !dbg_phase0_done && yfloor > 0) {
            dbg_phase0_done = true;
            atomicMax(F.dbg + 4, gtime_ns());      // end of phase 0 (Z + Y part 0) on this device
        }
        if (t >= total) break;
        if (F.dbg && threadIdx.x == 0) dbg_prev = gtime_ns();
        if (role == 0) {
            OpA::run(A, ka, (long long)plane * F.GA + idx, twa);
            __syncthreads();
            if (threadIdx.x == 0) {
                __threadfence();
                atomicAdd(F.plane_done + plane, 1ull);
            }
        } else if (role == 1) {
            if (threadIdx.x == 0) {
                unsigned long long v;
                SpinGuard guard;
                for (;;) {
                    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(F.plane_done + plane) : "memory");
                    if (v >= F.target) break;
                    __nanosleep(64);
                    guard.tick();
                }
            }
            __syncthreads();
            OpB::run(B, kb, (long long)plane * F.GB + (long long)part * F.GBk + idx, twb);
        } else {
            // the arrival of a part is polled once per CTA (arrived_mask, uniform): the acquire loads of threads 0..P-1 order
            // the senders' stores before everything after the bar.sync; no fence is needed on this side
            if (!((arrived_mask >> part) & 1u)) {
                if (threadIdx.x < F.P) {
                    const unsigned long long* flag = F.my_arrive + (size_t)part * DFFT_MAX_CHUNKS + threadIdx.x;
                    unsigned long long v;
                    SpinGuard guard;
                    for (;;) {
                        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flag) : "memory");
                        if (v >= F.epoch) break;
                        __nanosleep(128);
                        guard.tick();
                    }
                }
                arrived_mask |= 1u << part;
                __syncthreads();
                if (F.dbg && threadIdx.x == 0) { const unsigned long long now = gtime_ns(); dbg_wait += now - dbg_prev; dbg_prev = now; }
            }
            if (F.dbg && threadIdx.x == 0 && dbg_first_x) { dbg_first_x = false; atomicMin(F.dbg + 1, gtime_ns()); }
            const unsigned row = idx / (unsigned)F.GXk, bb = idx - row * (unsigned)F.GXk;
            OpC::run(Cc, kc, (long long)row * F.GX + (long long)part * F.GXk + bb, twc);
        }
        if (F.dbg && threadIdx.x == 0) { dbg_t[role] += gtime_ns() - dbg_prev; dbg_n[role]++; }
    }
    if (F.dbg && threadIdx.x == 0) {
        atomicMax(F.dbg + 5, gtime_ns());          // kernel end
        for (int r = 0; r < 3; r++) { atomicAdd(F.dbg + 6 + r, dbg_t[r]); atomicAdd(F.dbg + 9 + r, (unsigned long long)dbg_n[r]); }
        atomicAdd(F.dbg + 12, dbg_wait);
        atomicMax(F.dbg + 13, dbg_wait);
    }
    if (threadIdx.x == 0) {
        const unsigned left = atomicAdd(F.ticket + 1, 1u);
        if (left == gridDim.x - 1) { F.ticket[0] = 0; F.ticket[1] = 0; __threadfence(); }
    }
}

}  // namespace dfft
