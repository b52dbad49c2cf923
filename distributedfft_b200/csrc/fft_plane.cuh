// fft_plane.cuh -- the X and Y passes of a batched 3-D (or 2-D) transform over small square planes in ONE sweep.
//
// A CTA owns P whole n x n planes (P * n lines, at least 256 threads where the schedule allows).  Forward, per group of planes:
//   X role : the rows, loaded from global memory exactly as the contiguous pass (PK_Z, MAP_T) loads them, run through the
//            contiguous schedule with exchanges in shared memory; the results go into a shared-memory copy of the planes
//   Y role : the columns, read from that copy in the column-fastest map (MAP_C), run through the strided schedule and stored
//            as the strided pass (PK_Y) stores them -- adjacent threads hold adjacent x, so the stores are coalesced
// The inverse runs the Y role first (columns from global memory into a row-major copy), then the X role, with the swap
// convention of TileOp::run: swap on load, swap on store; the two swaps in between cancel and are left out.
//
// Results are bit-identical to the two separate passes: the entry's own schedules (the same Sched for both roles at the
// instantiated lengths), the same twiddle table, the same butterflies in the same order per line.  Twiddles are read from
// shared memory in both roles (the register copies of TileOp would differ per role's thread map); their values are the same.
//
// Every element of a group is in registers before any of it is stored, so in-place execution is safe; the plane copy and the
// exchange buffer are the same shared memory, separated by barriers:
//   - StageRunner (no ping-pong) synchronises before each scatter, so a role's first scatter waits for the previous readers;
//   - after the first role's last gather a barrier frees the buffer for the plane copy, and another one publishes the copy.
// Both roles use C = P * n lines of n points, so one line pitch SmemGeom::line(n, C) serves the exchanges and the copy.
// Shared memory: P * n padded lines + the twiddle table (64 x 64 fp64: 73 KB).
#pragma once
#include "fft_passes.cuh"

namespace dfft {

template <typename T> struct PlaneArgs {
    const cx<T>* in;
    cx<T>* out;
    const cx<T>* lut;      // the entry's twiddle table (Sched::lut_size() entries, shared by both roles)
    long long planes;      // densely packed n x n planes (row-major, x fastest)
    int inv;               // 1: inverse transform (e^{+i..}), unnormalised
};

template <class S, typename T, int P> struct PlaneSmem {
    static constexpr int C = P * S::N;
    static constexpr int LS = SmemGeom<T>::line(S::N, C);
    static constexpr size_t buf_bytes = ((size_t)C * LS * sizeof(cx<T>) + 15) / 16 * 16;
    static constexpr size_t lut_bytes = (size_t)((S::lut_size() * sizeof(cx<T>) + 15) / 16 * 16);
    static constexpr size_t bytes = buf_bytes + lut_bytes + 16;
};

// planes per CTA: the fewest whole planes that give at least 256 threads
template <class S> constexpr int plane_group() { return S::T * S::N >= 256 ? 1 : 256 / (S::T * S::N); }

template <class S, typename T, int P, int MINB>
__global__ void __launch_bounds__(S::T* S::N* P, MINB) fft_plane_kernel(const PlaneArgs<T> A)
{
    static_assert(S::valid() && S::NSTAGES > 1, "bad schedule");
    using SM = PlaneSmem<S, T, P>;
    constexpr int N = S::N, R = S::R, TT = S::T, C = SM::C, LS = SM::LS;
    constexpr long long NN = (long long)N * N;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    cx<T>* buf = reinterpret_cast<cx<T>*>(smem_raw);
    cx<T>* lut_s = reinterpret_cast<cx<T>*>(smem_raw + SM::buf_bytes);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + SM::buf_bytes + SM::lut_bytes);
    stage_twiddles_tma<T>(lut_s, A.lut, S::lut_size(), bar);

    const int tid = threadIdx.x;
    int tr, cr, tc, cc;   // row role: thread tr of line cr (MAP_T); column role: thread tc of column cc (MAP_C)
    thread_map<MAP_T, C, TT>(tid, tr, cr);
    thread_map<MAP_C, C, TT>(tid, tc, cc);
    const int pr = cr / N, yr = cr % N;   // row role: plane of the group and row y
    const int pc = cc / N, xc = cc % N;   // column role: plane of the group and column x
    const bool inv = A.inv != 0;
    const long long groups = (A.planes + P - 1) / P;
    cx<T> twr[1];
    int pp = 0;
    for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
        const long long p0 = g * P;
        const bool okr = p0 + pr < A.planes, okc = p0 + pc < A.planes;
        cx<T> v[R];
        if (!inv) {
            const cx<T>* src = A.in + (p0 + pr) * NN + (long long)yr * N + tr;
#pragma unroll
            for (int u = 0; u < R; u++) v[u] = okr ? ld_stream(src + u * TT) : mk<T>(0, 0);
            StageRunner<S, 0, T, C, MAP_T, MAP_T, false, false>::run(v, tr, cr, tr, cr, buf, pp, lut_s, twr, [] {});
            __syncthreads();   // every thread's last gather is done: the exchange buffer becomes the plane copy
            // point x = tr + u*TT of row yr -> column line (pr, x), position yr
#pragma unroll
            for (int u = 0; u < R; u++) buf[(pr * N + tr + u * TT) * LS + SmemGeom<T>::pad(yr)] = v[u];
            __syncthreads();
            stage_gather<S, T>(v, tc, buf + cc * LS);
            StageRunner<S, 0, T, C, MAP_C, MAP_C, false, false>::run(v, tc, cc, tc, cc, buf, pp, lut_s, twr, [] {});
            if (okc) {
                cx<T>* dst = A.out + (p0 + pc) * NN + (long long)tc * N + xc;
#pragma unroll
                for (int u = 0; u < R; u++) st_stream(dst + (long long)u * TT * N, v[u]);
            }
        } else {
            const cx<T>* src = A.in + (p0 + pc) * NN + (long long)tc * N + xc;
#pragma unroll
            for (int u = 0; u < R; u++) v[u] = okc ? cswap(ld_stream(src + (long long)u * TT * N)) : mk<T>(0, 0);
            StageRunner<S, 0, T, C, MAP_C, MAP_C, false, false>::run(v, tc, cc, tc, cc, buf, pp, lut_s, twr, [] {});
            __syncthreads();
            // point y = tc + u*TT of column xc -> row line (pc, y), position xc
#pragma unroll
            for (int u = 0; u < R; u++) buf[(pc * N + tc + u * TT) * LS + SmemGeom<T>::pad(xc)] = v[u];
            __syncthreads();
            stage_gather<S, T>(v, tr, buf + cr * LS);
            StageRunner<S, 0, T, C, MAP_T, MAP_T, false, false>::run(v, tr, cr, tr, cr, buf, pp, lut_s, twr, [] {});
            if (okr) {
                cx<T>* dst = A.out + (p0 + pr) * NN + (long long)yr * N + tr;
#pragma unroll
                for (int u = 0; u < R; u++) st_stream(dst + u * TT, cswap(v[u]));
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// fft_plane_conv_kernel -- a whole 2-D spectral convolution of small square images in ONE sweep: out = ifft2(fft2(in) * m)
// per image, unnormalised (x N*N) unless do_scale.  The CTA shape, thread maps and shared memory are fft_plane_kernel's; per
// group of P images:
//   X role forward  : rows (MAP_T) from global memory, contiguous schedule, column-line copy in shared memory
//   Y role forward  : columns (MAP_C) from the copy, strided schedule; thread (tc, cc) now holds y = tc + u*TT of column xc,
//                     its own load and store positions
//   multiply        : conv_tiles' expression, v = cswap(cmul(v, m)) (the inverse's swap-in folded into the product)
//   Y role inverse  : MAP_C, strided schedule (StageRunner's barrier before its first scatter frees the buffer)
//   X role inverse  : row-line copy, MAP_T, contiguous schedule, cswap on the store to the rows.  The XCONV pass's store swap
//                     and the inverse X pass's load swap of the separate passes cancel and are left out
// Bit-identical to the three passes X, XCONV along y, inverse X (DFFT_NO_PLANE=1): the same schedules and twiddle values (one
// Sched for both roles at the instantiated lengths), the same butterflies per line, the same multiply.  Every element of a
// group is in registers before any of it is stored (in place is safe); images past the batch load, read and store nothing.
// ------------------------------------------------------------------------------------------
template <typename T> struct PlaneConvArgs {
    PlaneArgs<T> p;        // p.planes = images; p.inv unused
    const cx<T>* mult;     // [images or 1][N][N], natural order
    long long mult_plane;  // multiplier elements between images: 0 (one multiplier for every image) or N*N
    T scale;               // folded into the multiplier when do_scale
    int do_scale;
};

template <class S, typename T, int P, int MINB>
__global__ void __launch_bounds__(S::T* S::N* P, MINB) fft_plane_conv_kernel(const PlaneConvArgs<T> R)
{
    static_assert(S::valid() && S::NSTAGES > 1, "bad schedule");
    using SM = PlaneSmem<S, T, P>;
    constexpr int N = S::N, RR = S::R, TT = S::T, C = SM::C, LS = SM::LS;
    constexpr long long NN = (long long)N * N;
    const PlaneArgs<T>& A = R.p;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    cx<T>* buf = reinterpret_cast<cx<T>*>(smem_raw);
    cx<T>* lut_s = reinterpret_cast<cx<T>*>(smem_raw + SM::buf_bytes);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + SM::buf_bytes + SM::lut_bytes);
    stage_twiddles_tma<T>(lut_s, A.lut, S::lut_size(), bar);

    const int tid = threadIdx.x;
    int tr, cr, tc, cc;   // row role: thread tr of line cr (MAP_T); column role: thread tc of column cc (MAP_C)
    thread_map<MAP_T, C, TT>(tid, tr, cr);
    thread_map<MAP_C, C, TT>(tid, tc, cc);
    const int pr = cr / N, yr = cr % N;   // row role: image of the group and row y
    const int pc = cc / N, xc = cc % N;   // column role: image of the group and column x
    const bool do_scale = R.do_scale != 0;
    const long long groups = (A.planes + P - 1) / P;
    cx<T> twr[1];
    int pp = 0;
    for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
        const long long p0 = g * P;
        const bool okr = p0 + pr < A.planes, okc = p0 + pc < A.planes;
        cx<T> v[RR];
        const cx<T>* src = A.in + (p0 + pr) * NN + (long long)yr * N + tr;
#pragma unroll
        for (int u = 0; u < RR; u++) v[u] = okr ? ld_stream(src + u * TT) : mk<T>(0, 0);
        StageRunner<S, 0, T, C, MAP_T, MAP_T, false, false>::run(v, tr, cr, tr, cr, buf, pp, lut_s, twr, [] {});
        __syncthreads();   // every thread's last gather is done: the exchange buffer becomes the image copy
        // point x = tr + u*TT of row yr -> column line (pr, x), position yr
#pragma unroll
        for (int u = 0; u < RR; u++) buf[(pr * N + tr + u * TT) * LS + SmemGeom<T>::pad(yr)] = v[u];
        __syncthreads();
        stage_gather<S, T>(v, tc, buf + cc * LS);
        StageRunner<S, 0, T, C, MAP_C, MAP_C, false, false>::run(v, tc, cc, tc, cc, buf, pp, lut_s, twr, [] {});
        const cx<T>* mp = R.mult + (p0 + pc) * R.mult_plane + (long long)tc * N + xc;
#pragma unroll
        for (int u = 0; u < RR; u++) {
            cx<T> m = okc ? ld_stream(mp + (long long)u * TT * N) : mk<T>(0, 0);
            if (do_scale) { m.x *= R.scale; m.y *= R.scale; }
            v[u] = cswap(cmul(v[u], m));
        }
        StageRunner<S, 0, T, C, MAP_C, MAP_C, false, false>::run(v, tc, cc, tc, cc, buf, pp, lut_s, twr, [] {});
        __syncthreads();
        // point y = tc + u*TT of column xc -> row line (pc, y), position xc
#pragma unroll
        for (int u = 0; u < RR; u++) buf[(pc * N + tc + u * TT) * LS + SmemGeom<T>::pad(xc)] = v[u];
        __syncthreads();
        stage_gather<S, T>(v, tr, buf + cr * LS);
        StageRunner<S, 0, T, C, MAP_T, MAP_T, false, false>::run(v, tr, cr, tr, cr, buf, pp, lut_s, twr, [] {});
        if (okr) {
            cx<T>* dst = A.out + (p0 + pr) * NN + (long long)yr * N + tr;
#pragma unroll
            for (int u = 0; u < RR; u++) st_stream(dst + u * TT, cswap(v[u]));
        }
    }
}

}  // namespace dfft
