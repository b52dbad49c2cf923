// fft_real.cuh -- the real-data Z passes of the R2C / C2R slab transforms.
//
// Two real lines a, b of length N are transformed as ONE complex line z = a + i b with the tuned N-point schedule of the
// C2C Z pass (TileOp's setup and twiddles, StageRunner's stages: nothing here changes the butterflies).  The two half spectra
// are then separated with the Hermitian symmetry of a real signal's transform, Z = FFT(z):
//   A[k] = (Z[k] + conj Z[(N-k) mod N]) / 2        = FFT(a)[k]
//   B[k] = (Z[k] - conj Z[(N-k) mod N]) / (2i)     = FFT(b)[k],   k = 0 .. N/2   (nzh = N/2 + 1 values, any N)
// and the inverse builds Z from the two half spectra, Z[k] = A[k] + i B[k] for k <= N/2 and conj A[N-k] + i conj B[N-k] above,
// runs the inverse schedule and stores Re z to line a and Im z to line b.  Like FFTW and numpy.fft.irfft, the inverse ignores
// the imaginary parts of A and B at k = 0 and (even N) k = N/2.
//
// Addressing: a tile is C line PAIRS.  Pair (tile, c) has its first line at  base + tile*SB + c*cs  and its second line `ld`
// elements further (real side in real elements, complex side in complex elements); the points of a line are contiguous
// (Affine::es must be 1).  TileArgs::W is the number of LINES: with an odd line count the last pair has no second line, which is
// then neither loaded nor stored.
#pragma once
#include "fft_passes.cuh"

namespace dfft {

template <typename T> struct RealZArgs {
    TileArgs<T> t;       // lut, ntiles, W (lines), inv, do_scale, scale; ia / oa: tile (SB) and pair (cs) strides of each side
    const T* rin;        // R2C: real input (C2R: t.in is the complex input)
    T* rout;             // C2R: real output (R2C: t.out is the complex output)
    long long ld_in, ld_out;   // distance between the two lines of a pair on the input / output side
};

// R2C: real lines -> half spectra (N/2 + 1 complex points per line)
template <class S, typename T, int C, bool TWREG, int MINB, bool PINGPONG>
__global__ void __launch_bounds__(S::T* C, MINB) fft_z_r2c_kernel(const RealZArgs<T> R)
{
    static_assert(S::valid() && S::NSTAGES > 1, "the split epilogue reuses the exchange buffer");
    using Op = TileOp<S, T, C, MAP_T, MAP_T, TWREG, false, false, PINGPONG>;
    constexpr int N = S::N, TT = S::T, NZH = N / 2 + 1, LS = SmemGeom<T>::line(N, C);
    const TileArgs<T>& A = R.t;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename Op::Ctx k;
    Op::setup(A, smem_raw, smem_raw + Op::SM::exch_bytes, k);
    cx<T> twr[Op::NTW];
    Op::load_twiddles(k, twr);
    const int t = k.t_in, c = k.c_in;   // MAP_T on both sides: t_out == t_in, c_out == c_in
    cx<T>* line = k.exch + c * LS;
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        const long long line0 = 2 * (tile * C + c);
        const bool oka = line0 < A.W, okb = line0 + 1 < A.W;
        const T* pa = R.rin + tile * A.ia.SB + c * A.ia.cs + t;
        const T* pb = pa + R.ld_in;
        cx<T> v[S::R];
#pragma unroll
        for (int u = 0; u < S::R; u++) v[u] = mk<T>(oka ? ld_stream(pa + u * TT) : (T)0, okb ? ld_stream(pb + u * TT) : (T)0);
        StageRunner<S, 0, T, C, MAP_T, MAP_T, TWREG, PINGPONG>::run(v, t, c, t, c, k.exch, k.pp, k.lut_s, twr, [] {});
        // Z[k] and Z[N-k] sit in different threads: through the exchange buffer (every thread is past its last gather)
        __syncthreads();
#pragma unroll
        for (int u = 0; u < S::R; u++) line[SmemGeom<T>::pad(t + u * TT)] = v[u];
        __syncthreads();
        cx<T>* qa = A.out + tile * A.oa.SB + c * A.oa.cs;
        cx<T>* qb = qa + R.ld_out;
        const T h = (T)0.5;
#pragma unroll
        for (int j0 = 0; j0 < NZH; j0 += TT) {
            const int j = j0 + t;
            if (j0 + TT <= NZH || j < NZH) {
                const cx<T> z = line[SmemGeom<T>::pad(j)], m = line[SmemGeom<T>::pad(j == 0 ? 0 : N - j)];
                if (oka) st_stream(qa + j, mk<T>(h * (z.x + m.x), h * (z.y - m.y)));
                if (okb) st_stream(qb + j, mk<T>(h * (z.y + m.y), h * (m.x - z.x)));
            }
        }
        __syncthreads();   // the next tile's first exchange reuses the buffer
    }
}

// C2R: half spectra -> real lines (unnormalised; TileArgs::do_scale multiplies by TileArgs::scale)
template <class S, typename T, int C, bool TWREG, int MINB, bool PINGPONG>
__global__ void __launch_bounds__(S::T* C, MINB) fft_z_c2r_kernel(const RealZArgs<T> R)
{
    static_assert(S::valid() && S::NSTAGES > 1, "bad schedule");
    using Op = TileOp<S, T, C, MAP_T, MAP_T, TWREG, false, false, PINGPONG>;
    constexpr int N = S::N, TT = S::T, NZH = N / 2 + 1;
    const TileArgs<T>& A = R.t;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename Op::Ctx k;
    Op::setup(A, smem_raw, smem_raw + Op::SM::exch_bytes, k);
    cx<T> twr[Op::NTW];
    Op::load_twiddles(k, twr);
    const int t = k.t_in, c = k.c_in;
    const T s = A.do_scale ? A.scale : (T)1;
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        const long long line0 = 2 * (tile * C + c);
        const bool oka = line0 < A.W, okb = line0 + 1 < A.W;
        const cx<T>* pa = A.in + tile * A.ia.SB + c * A.ia.cs;
        const cx<T>* pb = pa + R.ld_in;
        // z = A + i B below the middle, conj A + i conj B above, held swapped (re, im) for the inverse as in TileOp::run:
        // v = (Im z, Re z) = (A.y + B.x, A.x - B.y) below, (B.x - A.y, A.x + B.y) above.  Point e = t + u*TT reads j = e below
        // and j = N - e above; for every u but the one that straddles NZH the side is known at compile time, so the addresses
        // are a per-thread base plus an immediate.  Line a first, then line b: half the loads in flight at a time
        cx<T> v[S::R];
#pragma unroll
        for (int u = 0; u < S::R; u++) {
            const int e = t + u * TT;
            const bool mirror = (u + 1) * TT <= NZH ? false : (u * TT >= NZH ? true : e >= NZH);
            const int j = mirror ? N - e : e;
            cx<T> a = oka ? ld_stream(pa + j) : mk<T>(0, 0);
            if (!mirror && (j == 0 || 2 * j == N)) a.y = 0;
            v[u] = mk<T>(mirror ? -a.y : a.y, a.x);
        }
#pragma unroll
        for (int u = 0; u < S::R; u++) {
            const int e = t + u * TT;
            const bool mirror = (u + 1) * TT <= NZH ? false : (u * TT >= NZH ? true : e >= NZH);
            const int j = mirror ? N - e : e;
            cx<T> b = okb ? ld_stream(pb + j) : mk<T>(0, 0);
            if (!mirror && (j == 0 || 2 * j == N)) b.y = 0;
            v[u].x += b.x;
            v[u].y += mirror ? b.y : -b.y;
        }
        StageRunner<S, 0, T, C, MAP_T, MAP_T, TWREG, PINGPONG>::run(v, t, c, t, c, k.exch, k.pp, k.lut_s, twr, [] {});
        T* qa = R.rout + tile * A.oa.SB + c * A.oa.cs + t;
        T* qb = qa + R.ld_out;
#pragma unroll
        for (int u = 0; u < S::R; u++) {   // swapped back: Re z = v.y, Im z = v.x
            if (oka) st_stream(qa + u * TT, v[u].y * s);
            if (okb) st_stream(qb + u * TT, v[u].x * s);
        }
    }
}

}  // namespace dfft
