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

// 1-D convolution of real lines, real in / real out: out = irfft(rfft(in) * m, N) * N per line, in ONE pass (the 1-D R2C
// convolve lines plans).  The pair layout and loads of fft_z_r2c_kernel (z = a + i b, a missing second line reads 0), the forward
// stages, then Z goes through the exchange buffer so that every thread has the partner Z[(N-e) mod N] of each of its points e.
// Per point, with j = e for e <= N/2 and j = N - e above, and (F, G) = (Z[j], Z[N-j]) both read from {Z[e], partner}:
//   A = (F + conj G) / 2,  B = (F - conj G) / 2i          (the half spectra of lines a and b at j)
//   A' = A ma[j],  B' = B mb[j],  Im A' = Im B' = 0 at j = 0 and (even N) j = N/2   (the C2R convention of fft_z_c2r_kernel)
//   Z'[e] = A' + i B' for e <= N/2,  conj A' + i conj B' above
// and the inverse runs from cswap(Z') as in fft_z_c2r_kernel, Re z to line a, Im z to line b.  ma / mb: N/2 + 1 complex points
// at mult + line * mult_line (mult_line 0: one multiplier for every line).  Every element of a pair is in registers before any of
// it is stored, so in == out is safe.
template <typename T> struct RealLineConvArgs {
    RealZArgs<T> r;
    const cx<T>* mult;
    long long mult_line;   // multiplier elements between lines: 0 (one multiplier for every line) or N/2 + 1
};

template <class S, typename T, int C, bool TWREG, int MINB, bool PINGPONG>
__global__ void __launch_bounds__(S::T* C, MINB) fft_line_conv_r2c_kernel(const RealLineConvArgs<T> R)
{
    static_assert(S::valid() && S::NSTAGES > 1, "the pair split reuses the exchange buffer");
    using Op = TileOp<S, T, C, MAP_T, MAP_T, TWREG, false, false, PINGPONG>;
    constexpr int N = S::N, TT = S::T, LS = SmemGeom<T>::line(N, C);
    const TileArgs<T>& A = R.r.t;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename Op::Ctx k;
    Op::setup(A, smem_raw, smem_raw + Op::SM::exch_bytes, k);
    cx<T> twr[Op::NTW];
    Op::load_twiddles(k, twr);
    const int t = k.t_in, c = k.c_in;   // MAP_T on both sides: t_out == t_in, c_out == c_in
    cx<T>* line = k.exch + c * LS;
    const bool do_scale = A.do_scale != 0;
    const T h = (T)0.5;
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        const long long line0 = 2 * (tile * C + c);
        const bool oka = line0 < A.W, okb = line0 + 1 < A.W;
        const T* pa = R.r.rin + tile * A.ia.SB + c * A.ia.cs + t;
        const T* pb = pa + R.r.ld_in;
        cx<T> v[S::R];
#pragma unroll
        for (int u = 0; u < S::R; u++) v[u] = mk<T>(oka ? ld_stream(pa + u * TT) : (T)0, okb ? ld_stream(pb + u * TT) : (T)0);
        StageRunner<S, 0, T, C, MAP_T, MAP_T, TWREG, PINGPONG>::run(v, t, c, t, c, k.exch, k.pp, k.lut_s, twr, [] {});
        // Z[e] and Z[N-e] sit in different threads: through the exchange buffer (every thread is past its last gather)
        __syncthreads();
#pragma unroll
        for (int u = 0; u < S::R; u++) line[SmemGeom<T>::pad(t + u * TT)] = v[u];
        __syncthreads();
        const cx<T>* ma = R.mult + line0 * R.mult_line;
        const cx<T>* mb = ma + R.mult_line;
#pragma unroll
        for (int u = 0; u < S::R; u++) {
            const int e = t + u * TT;
            const bool mirror = 2 * e > N;
            const int j = mirror ? N - e : e;
            const cx<T> w = line[SmemGeom<T>::pad(e == 0 ? 0 : N - e)];
            const cx<T> f = mirror ? w : v[u], g = mirror ? v[u] : w;
            cx<T> xa = mk<T>(h * (f.x + g.x), h * (f.y - g.y)), xb = mk<T>(h * (f.y + g.y), h * (g.x - f.x));
            cx<T> fa = oka ? ld_stream(ma + j) : mk<T>(0, 0), fb = okb ? ld_stream(mb + j) : mk<T>(0, 0);
            if (do_scale) { fa.x *= A.scale; fa.y *= A.scale; fb.x *= A.scale; fb.y *= A.scale; }
            xa = cmul(xa, fa);
            xb = cmul(xb, fb);
            if (j == 0 || 2 * j == N) { xa.y = 0; xb.y = 0; }
            // cswap(Z'): (Im Z', Re Z') = (A'.y + B'.x, A'.x - B'.y) below, (B'.x - A'.y, A'.x + B'.y) above
            v[u] = mirror ? mk<T>(xb.x - xa.y, xa.x + xb.y) : mk<T>(xa.y + xb.x, xa.x - xb.y);
        }
        // every thread has read its partners before the inverse run's first scatter reuses the buffer
        __syncthreads();
        StageRunner<S, 0, T, C, MAP_T, MAP_T, TWREG, PINGPONG>::run(v, t, c, t, c, k.exch, k.pp, k.lut_s, twr, [] {});
        T* qa = R.r.rout + tile * A.oa.SB + c * A.oa.cs + t;
        T* qb = qa + R.r.ld_out;
#pragma unroll
        for (int u = 0; u < S::R; u++) {   // swapped back: Re z = v.y, Im z = v.x
            if (oka) st_stream(qa + u * TT, v[u].y);
            if (okb) st_stream(qb + u * TT, v[u].x);
        }
    }
}

}  // namespace dfft
