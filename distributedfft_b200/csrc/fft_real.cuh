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

// The per-point step of the real convolutions, shared by fft_line_conv_r2c_kernel (and its padded twin) and fft_conv_r2c_kernel:
// (F, G) = (f, g) = (Z[j], Z[n-j]) of z = a + i b at j = min(e, n - e), `mirror` = (e > n/2), `edge` = (j == 0 or 2j == n); the
// multipliers ma[j], mb[j] of lines a and b, read where oka / okb (else 0), times `scale` when do_scale.  Sets v = cswap(Z'[e]), the
// first value of the inverse run.  A statement macro, not a __forceinline__ function: the function's locals, spliced into the
// kernel at inlining, renumbered fft_line_conv_r2c_kernel's registers (+2 at 49 fp64, 24 B more spill at 243 fp64 under
// -Xptxas -v); expanded in place the kernel compiles exactly as it did with the statements written out.
#define DFFT_R2C_CONV_POINT(T, v, f_, g_, mirror, edge, ma, mb, j, oka, okb, do_scale, scale)                                        \
    do {                                                                                                                             \
        const cx<T> f = f_, g = g_;                                                                                                  \
        cx<T> xa = mk<T>((T)0.5 * (f.x + g.x), (T)0.5 * (f.y - g.y)), xb = mk<T>((T)0.5 * (f.y + g.y), (T)0.5 * (g.x - f.x));       \
        cx<T> fa = (oka) ? ld_stream((ma) + (j)) : mk<T>(0, 0), fb = (okb) ? ld_stream((mb) + (j)) : mk<T>(0, 0);                   \
        if (do_scale) { fa.x *= (scale); fa.y *= (scale); fb.x *= (scale); fb.y *= (scale); }                                      \
        xa = cmul(xa, fa);                                                                                                           \
        xb = cmul(xb, fb);                                                                                                           \
        if (edge) { xa.y = 0; xb.y = 0; }                                                                                            \
        /* cswap(Z'): (Im Z', Re Z') = (A'.y + B'.x, A'.x - B'.y) below, (B'.x - A'.y, A'.x + B'.y) above */                        \
        v = (mirror) ? mk<T>(xb.x - xa.y, xa.x + xb.y) : mk<T>(xa.y + xb.x, xa.x - xb.y);                                          \
    } while (0)

// PAD (fft_line_conv_pad_r2c_kernel): point e of a line loads only where e < in_len and stores only where e < out_len
template <class S, typename T, int C, bool TWREG, bool PINGPONG, bool PAD>
__device__ __forceinline__ void line_conv_r2c_tiles(const RealLineConvArgs<T>& R, long long in_len, long long out_len)
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
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        const long long line0 = 2 * (tile * C + c);
        const bool oka = line0 < A.W, okb = line0 + 1 < A.W;
        const T* pa = R.r.rin + tile * A.ia.SB + c * A.ia.cs + t;
        const T* pb = pa + R.r.ld_in;
        cx<T> v[S::R];
#pragma unroll
        for (int u = 0; u < S::R; u++) {
            const bool in = !PAD || t + u * TT < in_len;
            v[u] = mk<T>(oka && in ? ld_stream(pa + u * TT) : (T)0, okb && in ? ld_stream(pb + u * TT) : (T)0);
        }
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
            DFFT_R2C_CONV_POINT(T, v[u], mirror ? w : v[u], mirror ? v[u] : w, mirror, j == 0 || 2 * j == N, ma, mb, j, oka, okb, do_scale, A.scale);
        }
        // every thread has read its partners before the inverse run's first scatter reuses the buffer
        __syncthreads();
        StageRunner<S, 0, T, C, MAP_T, MAP_T, TWREG, PINGPONG>::run(v, t, c, t, c, k.exch, k.pp, k.lut_s, twr, [] {});
        T* qa = R.r.rout + tile * A.oa.SB + c * A.oa.cs + t;
        T* qb = qa + R.r.ld_out;
#pragma unroll
        for (int u = 0; u < S::R; u++) {   // swapped back: Re z = v.y, Im z = v.x
            if (PAD && t + u * TT >= out_len) continue;
            if (oka) st_stream(qa + u * TT, v[u].y);
            if (okb) st_stream(qb + u * TT, v[u].x);
        }
    }
}

template <class S, typename T, int C, bool TWREG, int MINB, bool PINGPONG>
__global__ void __launch_bounds__(S::T* C, MINB) fft_line_conv_r2c_kernel(const RealLineConvArgs<T> R)
{
    line_conv_r2c_tiles<S, T, C, TWREG, PINGPONG, false>(R, 0, 0);
}

// RealPadArgs: the real padded kinds' arguments (the real zero-padded convolve lines plan).  A real line of `in` holds in_len points
// and one of `out` out_len (PadArgs' meaning).  `lines` counts the caller's real lines: the four-step kinds' TileArgs::W counts
// columns, and the last pair of an odd count has no second line
template <typename T> struct RealPadArgs {
    RealLineConvArgs<T> c;   // tile arguments, real lines and pair distances, multiplier
    long long in_len, out_len;
    long long lines;
};

// the short path of the real zero-padded 1-D convolve lines plans: fft_line_conv_r2c_kernel over lines of in_len points in,
// out_len out (LINE_CONV_PAD_R2C)
template <class S, typename T, int C, bool TWREG, int MINB, bool PINGPONG>
__global__ void __launch_bounds__(S::T* C, MINB) fft_line_conv_pad_r2c_kernel(const RealPadArgs<T> P)
{
    line_conv_r2c_tiles<S, T, C, TWREG, PINGPONG, true>(P.c, P.in_len, P.out_len);
}

// ------------------------------------------------------------------------------------------
// The middle pass of the real plan's long path (XCONV_R2C): the column convolve of n2 = S::N over the temporary [n2][n1] of each
// line pair (z = a + i b, written by XF_TW_PAD_R2C), in place, with the pair untangled around the multiply.  MAP_C on both sides,
// TileArgs as PK_XCONV's (W = n1 column positions per row); column position cp holds column k1 with mirror_pos<n1>(k1) = cp.
// After the forward run along n2, element (row k2, column k1) is Z[e], e = k1 + n1 k2, and its mirror Z[n - e] is element
//   (n2 - 1 - k2, n1 - k1) for k1 != 0: the other column of cp's aligned position pair (cp ^ 1), or cp itself when 2 k1 = n1
//   ((n2 - k2) mod n2, 0) for k1 == 0
// C is even, so a tile (columns b*C ... b*C + C - 1) holds whole mirror sets, a partial last tile included.  Through the exchange
// buffer every thread reads the partner of each of its elements, DFFT_R2C_CONV_POINT forms cswap(Z'), the inverse run along n2 follows
// and the result is stored back in place (the swapped-back value, as PK_XCONV stores).  ma / mb: n/2 + 1 points of lines 2a and
// 2a + 1 at mult + 2a * mult_line (mult_line 0: one multiplier for every line); a missing second line reads no multiplier.
// Unnormalised; TileArgs::do_scale folds TileArgs::scale into the multiply.
// ------------------------------------------------------------------------------------------
template <class S, typename T, int C, bool TWREG, int MINB, bool PINGPONG>
__global__ void __launch_bounds__(S::T* C, MINB) fft_conv_r2c_kernel(const RealPadArgs<T> P)
{
    static_assert(S::valid() && S::NSTAGES > 1, "the mirror exchange reuses the exchange buffer");
    static_assert(C % 2 == 0, "a tile must hold whole mirror pairs of columns");
    using Op = TileOp<S, T, C, MAP_C, MAP_C, TWREG, false, false, PINGPONG>;
    constexpr int RR = S::R, TT = S::T, N2 = S::N, LS = SmemGeom<T>::line(N2, C);
    const TileArgs<T>& A = P.c.r.t;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typename Op::Ctx k;
    Op::setup(A, smem_raw, smem_raw + Op::SM::exch_bytes, k);
    cx<T> twr[Op::NTW];
    Op::load_twiddles(k, twr);
    const int t = k.t_in, c = k.c_in;   // MAP_C on both sides: t_out == t_in, c_out == c_in
    const int n1 = A.W, n = n1 * N2;
    const bool do_scale = A.do_scale != 0;
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        const long long a = tile / A.G;
        const int b = (int)(tile - a * A.G);
        const int cp = b * C + c;
        const bool ok = cp < A.W, okb = 2 * a + 1 < P.lines;
        const int k1 = n1 % 2 ? (cp == n1 - 1 ? 0 : (cp % 2 ? n1 - (cp + 1) / 2 : cp / 2 + 1)) : (cp < 2 ? cp * (n1 / 2) : (cp % 2 ? n1 - cp / 2 : cp / 2));
        const bool self = k1 == 0 || 2 * k1 == n1;
        const long long off = a * A.ia.SA + b * A.ia.SB + c * A.ia.cs + (long long)t * A.ia.es;
        cx<T> v[RR];
#pragma unroll
        for (int u = 0; u < RR; u++) v[u] = ok ? ld_stream(A.in + off + (long long)u * TT * A.ia.es) : mk<T>(0, 0);
        StageRunner<S, 0, T, C, MAP_C, MAP_C, TWREG, PINGPONG>::run(v, t, c, t, c, k.exch, k.pp, k.lut_s, twr, [] {});
        // the partners sit in other threads: through the exchange buffer (every thread is past its last gather)
        __syncthreads();
#pragma unroll
        for (int u = 0; u < RR; u++) k.exch[c * LS + SmemGeom<T>::pad(t + u * TT)] = v[u];
        __syncthreads();
        const cx<T>* partner = k.exch + (self ? c : c ^ 1) * LS;
        const cx<T>* ma = P.c.mult + 2 * a * P.c.mult_line;
        const cx<T>* mb = ma + P.c.mult_line;
#pragma unroll
        for (int u = 0; u < RR; u++) {
            const int k2 = t + u * TT;
            const int e = k1 + n1 * k2;
            const bool mirror = 2 * e > n;
            const int j = mirror ? n - e : e;
            const cx<T> w = partner[SmemGeom<T>::pad(k1 ? N2 - 1 - k2 : (k2 ? N2 - k2 : 0))];
            DFFT_R2C_CONV_POINT(T, v[u], mirror ? w : v[u], mirror ? v[u] : w, mirror, j == 0 || 2 * j == n, ma, mb, j, ok, ok && okb, do_scale, A.scale);
        }
        // every thread has read its partners before the inverse run's first scatter reuses the buffer
        __syncthreads();
        StageRunner<S, 0, T, C, MAP_C, MAP_C, TWREG, PINGPONG>::run(v, t, c, t, c, k.exch, k.pp, k.lut_s, twr, [] {});
        if (ok) {
            cx<T>* q = A.out + a * A.oa.SA + b * A.oa.SB + c * A.oa.cs + (long long)t * A.oa.es;
#pragma unroll
            for (int u = 0; u < RR; u++) st_stream(q + (long long)u * TT * A.oa.es, cswap(v[u]));
        }
    }
}

}  // namespace dfft
