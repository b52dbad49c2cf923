// fft_generic.cuh -- run-time-scheduled pass kernel for transform lengths that have no tuned
// instantiation: any N whose prime factors are in {2,3,5,7,11,13} -- the set templateFFT accepts
// (templateFFT/src/templateFFT.cpp:3956-3964 factors N over 2..13 and rejects the rest) -- as long as
// one tile of two ping-pong lines fits in shared memory.
//
// Same tile/affine/chunk-table addressing and the same Stockham stage formulas as fft_tile_kernel
// (fft_passes.cuh), but the radix list is data, every stage goes through shared memory, and a thread
// keeps only one butterfly in registers at a time.  Slower than the tuned kernels (no register-resident
// stages, unpadded exchange buffers) -- it exists for API parity, not for the headline sizes.
#pragma once
#include "fft_passes.cuh"
#include "fft_real.cuh"

namespace dfft {

constexpr int GEN_MAX_STAGES = 24;
constexpr int GEN_THREADS = 256;

struct GenSched {
    int N, nstages, C;
    int rad[GEN_MAX_STAGES];
    int ns[GEN_MAX_STAGES];        // product of the radices before stage s
    int lut_off[GEN_MAX_STAGES];   // offset of stage s in the twiddle table (layout of build_lut)
};

// e^{-2 pi i t/p} for the two prime radices without a hand-written butterfly
template <typename T> __device__ __forceinline__ cx<T> prime_root(int p, int t)
{
    const double c11[11] = {1.0, 0.8412535328311811688618, 0.4154150130018864255292, -0.142314838273285140443, -0.654860733945285064056,
                            -0.959492973614497389890, -0.959492973614497389890, -0.654860733945285064056, -0.142314838273285140443,
                            0.4154150130018864255292, 0.8412535328311811688618};
    const double s11[11] = {0.0, 0.5406408174555975821076, 0.9096319953545183714117, 0.9898214418809327323760, 0.7557495743542582837740,
                            0.2817325568414296977114, -0.281732556841429697711, -0.755749574354258283774, -0.989821441880932732376,
                            -0.909631995354518371411, -0.540640817455597582107};
    const double c13[13] = {1.0, 0.8854560256532098959003, 0.5680647467311558025118, 0.1205366802553230533490, -0.354604887042535625969,
                            -0.748510748171101098634, -0.970941817426052027156, -0.970941817426052027156, -0.748510748171101098634,
                            -0.354604887042535625969, 0.1205366802553230533490, 0.5680647467311558025118, 0.8854560256532098959003};
    const double s13[13] = {0.0, 0.4647231720437685456560, 0.8229838658936563945796, 0.9927088740980539928007, 0.9350162426854148234397,
                            0.6631226582407952023767, 0.2393156642875577671487, -0.239315664287557767148, -0.663122658240795202376,
                            -0.935016242685414823439, -0.992708874098053992800, -0.822983865893656394579, -0.464723172043768545656};
    return p == 11 ? mk<T>((T)c11[t], (T)-s11[t]) : mk<T>((T)c13[t], (T)-s13[t]);
}

// forward DFT of prime length P (11 or 13) on registers v[0..P), O(P^2); fully unrolled so the root indices fold
template <typename T, int P> __device__ __forceinline__ void bfly_prime(cx<T>* v)
{
    cx<T> out[P];
#pragma unroll
    for (int q = 0; q < P; q++) {
        cx<T> acc = v[0];
#pragma unroll
        for (int m = 1; m < P; m++) acc = cadd(acc, cmul(v[m], prime_root<T>(P, (q * m) % P)));
        out[q] = acc;
    }
#pragma unroll
    for (int q = 0; q < P; q++) v[q] = out[q];
}

// all butterflies of one stage of radix R: item i = (line c, butterfly j); inputs src[c][j + m*NB],
// twiddle k = j mod NS, outputs dst[c][(j-k)*R + k + m*NS]  (the formulas of stage_scatter in fft_core.cuh)
template <typename T, int R>
__device__ __forceinline__ void generic_stage(const cx<T>* src, cx<T>* dst, const cx<T>* __restrict__ lut, int N, int C, int NS, bool tw)
{
    const int NB = N / R;
    for (int i = threadIdx.x; i < C * NB; i += GEN_THREADS) {
        const int j = i % NB, c = i / NB;
        const int k = j % NS;
        cx<T> v[R];
        const cx<T>* sp = src + c * N + j;
#pragma unroll
        for (int m = 0; m < R; m++) v[m] = sp[m * NB];
        if (tw) {
#pragma unroll
            for (int m = 1; m < R; m++) v[m] = cmul(v[m], __ldg(lut + (m - 1) * NS + k));
        }
        if constexpr (R == 11 || R == 13) bfly_prime<T, R>(v);
        else bfly<R, T, 1>(v);
        cx<T>* dp = dst + c * N + (j - k) * R + k;
#pragma unroll
        for (int m = 0; m < R; m++) dp[m * NS] = v[m];
    }
}

// MAPIN/MAPOUT only choose which index runs fastest across threads when the tile is moved between
// global and shared memory (MAP_T: along the line, MAP_C: across the C lines), i.e. coalescing.
template <typename T, int MAPIN, int MAPOUT, bool CHUNK_IN, bool CHUNK_OUT>
__global__ void __launch_bounds__(GEN_THREADS) fft_generic_kernel(const TileArgs<T> A, const GenSched G)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int N = G.N, C = G.C;
    cx<T>* buf0 = reinterpret_cast<cx<T>*>(smem_raw);
    cx<T>* buf1 = buf0 + (size_t)C * N;
    const int tid = threadIdx.x;
    const bool inv = A.inv != 0;
    const int total = C * N;

    wait_flags_at_start<T>(A);
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        const long long a = tile / A.G;
        const int b = (int)(tile - a * A.G);
        const int valid = min(C, A.W - b * C);   // lines of this tile that exist
        __syncthreads();                          // the previous tile's stores have read buf
        // ---- global -> shared (line c, point e at buf0[c*N + e])
        for (int i = tid; i < total; i += GEN_THREADS) {
            int c, e;
            if (MAPIN == MAP_T) { e = i % N; c = i / N; } else { c = i % C; e = i / C; }
            cx<T> v = mk<T>(0, 0);
            if (c < valid) {
                const cx<T>* p;
                if constexpr (!CHUNK_IN) p = A.in + a * A.ia.SA + b * A.ia.SB + c * A.ia.cs + (long long)e * A.ia.es;
                else {
                    int q = e / A.ci.ediv;
                    q = q < A.ci.nchunks ? q : A.ci.nchunks - 1;
                    p = reinterpret_cast<const cx<T>*>(A.ci.cptr[q]) + a * A.ci.SAq[q] + b * A.ia.SB + c * A.ia.cs + (long long)(e - q * A.ci.ediv) * A.ia.es;
                }
                v = ld_stream(p);
                if (inv) v = cswap(v);
            }
            buf0[c * N + e] = v;
        }
        __syncthreads();
        // ---- Stockham stages, ping-pong between the two buffers
        cx<T>* src = buf0;
        cx<T>* dst = buf1;
        for (int s = 0; s < G.nstages; s++) {
            const int NS = G.ns[s];
            const cx<T>* lut = A.lut + G.lut_off[s];
            switch (G.rad[s]) {
                case 2: generic_stage<T, 2>(src, dst, lut, N, C, NS, s > 0); break;
                case 3: generic_stage<T, 3>(src, dst, lut, N, C, NS, s > 0); break;
                case 4: generic_stage<T, 4>(src, dst, lut, N, C, NS, s > 0); break;
                case 5: generic_stage<T, 5>(src, dst, lut, N, C, NS, s > 0); break;
                case 7: generic_stage<T, 7>(src, dst, lut, N, C, NS, s > 0); break;
                case 8: generic_stage<T, 8>(src, dst, lut, N, C, NS, s > 0); break;
                case 11: generic_stage<T, 11>(src, dst, lut, N, C, NS, s > 0); break;
                case 13: generic_stage<T, 13>(src, dst, lut, N, C, NS, s > 0); break;
                default: __trap();
            }
            __syncthreads();
            cx<T>* t = src; src = dst; dst = t;
        }
        // ---- shared -> global (result in src)
        for (int i = tid; i < total; i += GEN_THREADS) {
            int c, e;
            if (MAPOUT == MAP_T) { e = i % N; c = i / N; } else { c = i % C; e = i / C; }
            if (c >= valid) continue;
            cx<T> v = src[c * N + e];
            if (A.tw_n) v = cmul(v, unit_root<T>((((long long)b * C + c) * (long long)e) % A.tw_n, A.tw_n));   // four-step twiddle
            if (inv) v = cswap(v);
            if (A.do_scale) { v.x *= A.scale; v.y *= A.scale; }
            cx<T>* p;
            if constexpr (!CHUNK_OUT) p = A.out + a * A.oa.SA + b * A.oa.SB + c * A.oa.cs + (long long)e * A.oa.es;
            else {
                int q = e / A.co.ediv;
                q = q < A.co.nchunks ? q : A.co.nchunks - 1;
                p = reinterpret_cast<cx<T>*>(A.co.cptr[q]) + a * A.co.SAq[q] + b * A.oa.SB + c * A.oa.cs + (long long)(e - q * A.co.ediv) * A.oa.es;
            }
            st_stream(p, v);
        }
    }
    signal_when_grid_done<T>(A);
}

// ------------------------------------------------------------------------------------------------
// Real-data passes on the run-time schedule: the generic counterparts of fft_z_r2c_kernel / fft_z_c2r_kernel (fft_real.cuh),
// same RealZArgs addressing (a tile is C line PAIRS, pair (tile, c) at base + tile*SB + c*cs, its second line `ld` further,
// TileArgs::W = number of lines, points contiguous) and the same split formulas.  A pair occupies one line of each ping-pong
// buffer, so the shared-memory footprint is that of fft_generic_kernel with the same C.

// every stage of G on C lines starting in buf0; returns the buffer that holds the result
template <typename T>
__device__ __forceinline__ cx<T>* generic_stages(cx<T>* buf0, cx<T>* buf1, const cx<T>* __restrict__ lut0, const GenSched& G)
{
    cx<T>* src = buf0;
    cx<T>* dst = buf1;
    for (int s = 0; s < G.nstages; s++) {
        const int NS = G.ns[s];
        const cx<T>* lut = lut0 + G.lut_off[s];
        switch (G.rad[s]) {
            case 2: generic_stage<T, 2>(src, dst, lut, G.N, G.C, NS, s > 0); break;
            case 3: generic_stage<T, 3>(src, dst, lut, G.N, G.C, NS, s > 0); break;
            case 4: generic_stage<T, 4>(src, dst, lut, G.N, G.C, NS, s > 0); break;
            case 5: generic_stage<T, 5>(src, dst, lut, G.N, G.C, NS, s > 0); break;
            case 7: generic_stage<T, 7>(src, dst, lut, G.N, G.C, NS, s > 0); break;
            case 8: generic_stage<T, 8>(src, dst, lut, G.N, G.C, NS, s > 0); break;
            case 11: generic_stage<T, 11>(src, dst, lut, G.N, G.C, NS, s > 0); break;
            case 13: generic_stage<T, 13>(src, dst, lut, G.N, G.C, NS, s > 0); break;
            default: __trap();
        }
        __syncthreads();
        cx<T>* t = src; src = dst; dst = t;
    }
    return src;
}

// R2C: z = a + i b per pair, the stages, then A / B straight from the transformed line in shared memory
template <typename T>
__global__ void __launch_bounds__(GEN_THREADS) fft_generic_r2c_kernel(const RealZArgs<T> R, const GenSched G)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const TileArgs<T>& A = R.t;
    const int N = G.N, C = G.C, H = N / 2 + 1;
    cx<T>* buf0 = reinterpret_cast<cx<T>*>(smem_raw);
    cx<T>* buf1 = buf0 + (size_t)C * N;
    const int tid = threadIdx.x;
    const T h = (T)0.5;
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        __syncthreads();                          // the previous tile's split has read its result buffer
        for (int i = tid; i < C * N; i += GEN_THREADS) {   // threads along the line: coalesced
            const int e = i % N, c = i / N;
            const long long line0 = 2 * (tile * C + c);
            const T* pa = R.rin + tile * A.ia.SB + c * A.ia.cs + e;
            buf0[i] = mk<T>(line0 < A.W ? ld_stream(pa) : (T)0, line0 + 1 < A.W ? ld_stream(pa + R.ld_in) : (T)0);
        }
        __syncthreads();
        const cx<T>* z = generic_stages<T>(buf0, buf1, A.lut, G);
        for (int i = tid; i < C * H; i += GEN_THREADS) {
            const int j = i % H, c = i / H;
            const long long line0 = 2 * (tile * C + c);
            if (line0 >= A.W) continue;
            const cx<T> p = z[c * N + j], m = z[c * N + (j == 0 ? 0 : N - j)];
            cx<T>* qa = A.out + tile * A.oa.SB + c * A.oa.cs + j;
            st_stream(qa, mk<T>(h * (p.x + m.x), h * (p.y - m.y)));
            if (line0 + 1 < A.W) st_stream(qa + R.ld_out, mk<T>(h * (p.y + m.y), h * (m.x - p.x)));
        }
    }
}

// C2R: Z = A + i B up to N/2, conj A[N-j] + i conj B[N-j] above (Im A, Im B dropped at j = 0 and, even N, j = N/2), loaded
// swapped as in fft_generic_kernel's inverse; after the stages Re z = v.y goes to line a and Im z = v.x to line b
template <typename T>
__global__ void __launch_bounds__(GEN_THREADS) fft_generic_c2r_kernel(const RealZArgs<T> R, const GenSched G)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const TileArgs<T>& A = R.t;
    const int N = G.N, C = G.C, H = N / 2 + 1;
    cx<T>* buf0 = reinterpret_cast<cx<T>*>(smem_raw);
    cx<T>* buf1 = buf0 + (size_t)C * N;
    const int tid = threadIdx.x;
    const T s = A.do_scale ? A.scale : (T)1;
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        __syncthreads();                          // the previous tile's stores have read its result buffer
        for (int i = tid; i < C * N; i += GEN_THREADS) {
            const int e = i % N, c = i / N;
            const long long line0 = 2 * (tile * C + c);
            const bool mirror = e >= H;
            const int j = mirror ? N - e : e;
            const cx<T>* pa = A.in + tile * A.ia.SB + c * A.ia.cs + j;
            cx<T> a = line0 < A.W ? ld_stream(pa) : mk<T>(0, 0);
            cx<T> b = line0 + 1 < A.W ? ld_stream(pa + R.ld_in) : mk<T>(0, 0);
            if (j == 0 || 2 * j == N) { a.y = 0; b.y = 0; }
            // z = (a.x - b.y, a.y + b.x) below, (a.x + b.y, b.x - a.y) above; stored as (Im z, Re z)
            buf0[i] = mirror ? mk<T>(b.x - a.y, a.x + b.y) : mk<T>(a.y + b.x, a.x - b.y);
        }
        __syncthreads();
        const cx<T>* z = generic_stages<T>(buf0, buf1, A.lut, G);
        for (int i = tid; i < C * N; i += GEN_THREADS) {
            const int e = i % N, c = i / N;
            const long long line0 = 2 * (tile * C + c);
            if (line0 >= A.W) continue;
            const cx<T> v = z[i];
            T* qa = R.rout + tile * A.oa.SB + c * A.oa.cs + e;
            st_stream(qa, v.y * s);
            if (line0 + 1 < A.W) st_stream(qa + R.ld_out, v.x * s);
        }
    }
}

}  // namespace dfft
