// fft_core.cuh -- in-register Stockham radix butterflies and the stage/exchange machinery shared
// by the three pass kernels (Z contiguous, Y strided + fused pack, X strided + fused unpack and
// transposed store).  Hand-written for sm_90a; no library FFT anywhere on this path.
//
// What this replaces in the reference: the hiprtc-generated `FFT_main` kernels of templateFFT
// (templateFFT/src/templateFFT.cpp:4699-4996 shaderGenFFT; radix butterflies :315-1075
// inlineRadixKernelFFT; smem shuffle :2466 appendRadixShuffle).  The maths is the same
// Stockham autosort decomposition; the code is not generated at run time but instantiated
// from templates for each supported (length, registers/thread, radix list).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dfft {

// ------------------------------------------------------------------------------------------
// complex helpers
// ------------------------------------------------------------------------------------------
template <typename T> struct cxt;
template <> struct cxt<double> { using type = double2; };
template <> struct cxt<float> { using type = float2; };
template <typename T> using cx = typename cxt<T>::type;

template <typename T> __device__ __forceinline__ cx<T> mk(T a, T b) { cx<T> r; r.x = a; r.y = b; return r; }
template <typename C> __device__ __forceinline__ C cadd(C a, C b) { a.x += b.x; a.y += b.y; return a; }
template <typename C> __device__ __forceinline__ C csub(C a, C b) { a.x -= b.x; a.y -= b.y; return a; }
// a * b, 2 mul + 2 fma
template <typename C> __device__ __forceinline__ C cmul(C a, C b)
{
    C r;
    r.x = fma(-a.y, b.y, a.x * b.x);
    r.y = fma(a.x, b.y, a.y * b.x);
    return r;
}
// a * (-i)
template <typename C> __device__ __forceinline__ C mul_mi(C a) { C r; r.x = a.y; r.y = -a.x; return r; }
// swap re<->im : IFFT(x) = swap(FFT(swap(x))), so the inverse transform reuses the forward code
template <typename C> __device__ __forceinline__ C cswap(C a) { C r; r.x = a.y; r.y = a.x; return r; }

// ------------------------------------------------------------------------------------------
// forward (e^{-i...}) small DFTs on registers v[0], v[S], v[2S], ... ; natural output order
// ------------------------------------------------------------------------------------------
template <typename T, int S> __device__ __forceinline__ void bfly2(cx<T>* v)
{
    cx<T> a = v[0], b = v[S];
    v[0] = cadd(a, b);
    v[S] = csub(a, b);
}

template <typename T, int S> __device__ __forceinline__ void bfly4(cx<T>* v)
{
    cx<T> s0 = cadd(v[0], v[2 * S]), s1 = csub(v[0], v[2 * S]);
    cx<T> s2 = cadd(v[S], v[3 * S]), s3 = mul_mi(csub(v[S], v[3 * S]));
    v[0] = cadd(s0, s2);
    v[S] = cadd(s1, s3);
    v[2 * S] = csub(s0, s2);
    v[3 * S] = csub(s1, s3);
}

template <typename T, int S> __device__ __forceinline__ void bfly8(cx<T>* v)
{
    const T h = (T)0.70710678118654752440084436210485;
    // decimation in frequency: even outputs = DFT4(x[n]+x[n+4]), odd = DFT4((x[n]-x[n+4]) W8^n)
    cx<T> a0 = cadd(v[0], v[4 * S]), b0 = csub(v[0], v[4 * S]);
    cx<T> a1 = cadd(v[S], v[5 * S]), d1 = csub(v[S], v[5 * S]);
    cx<T> a2 = cadd(v[2 * S], v[6 * S]), b2 = mul_mi(csub(v[2 * S], v[6 * S]));
    cx<T> a3 = cadd(v[3 * S], v[7 * S]), d3 = csub(v[3 * S], v[7 * S]);
    cx<T> b1 = mk<T>((d1.x + d1.y) * h, (d1.y - d1.x) * h);    // * (1-i)/sqrt2
    cx<T> b3 = mk<T>((d3.y - d3.x) * h, -(d3.x + d3.y) * h);   // * (-1-i)/sqrt2
    {
        cx<T> s0 = cadd(a0, a2), s1 = csub(a0, a2), s2 = cadd(a1, a3), s3 = mul_mi(csub(a1, a3));
        v[0] = cadd(s0, s2);
        v[2 * S] = cadd(s1, s3);
        v[4 * S] = csub(s0, s2);
        v[6 * S] = csub(s1, s3);
    }
    {
        cx<T> s0 = cadd(b0, b2), s1 = csub(b0, b2), s2 = cadd(b1, b3), s3 = mul_mi(csub(b1, b3));
        v[S] = cadd(s0, s2);
        v[3 * S] = cadd(s1, s3);
        v[5 * S] = csub(s0, s2);
        v[7 * S] = csub(s1, s3);
    }
}

template <typename T, int S> __device__ __forceinline__ void bfly16(cx<T>* v)
{
    // 16 = 4 x 4: n = n1 + 4 n2, k = 4 k1 + k2.  DFT4 over n2 (stride 4S), twiddle W16^(n1 k2),
    // DFT4 over n1 (stride S) -> result for k = k2 + 4 k1 sits at slot n2'=k2... we then place
    // it in natural order.
    const T c1 = (T)0.92387953251128675612818318939679;  // cos(pi/8)
    const T s1 = (T)0.38268343236508977172845998403040;  // sin(pi/8)
    const T h = (T)0.70710678118654752440084436210485;
#pragma unroll
    for (int n1 = 0; n1 < 4; n1++) bfly4<T, 4 * S>(v + n1 * S);  // slot (n1 + 4 k2) now holds sum over n2
    // twiddles W16^(n1*k2), W16 = e^{-i pi/8}
    v[(1 + 4 * 1) * S] = cmul(v[(1 + 4 * 1) * S], mk<T>(c1, -s1));   // W^1
    v[(1 + 4 * 2) * S] = cmul(v[(1 + 4 * 2) * S], mk<T>(h, -h));     // W^2
    v[(1 + 4 * 3) * S] = cmul(v[(1 + 4 * 3) * S], mk<T>(s1, -c1));   // W^3
    v[(2 + 4 * 1) * S] = cmul(v[(2 + 4 * 1) * S], mk<T>(h, -h));     // W^2
    v[(2 + 4 * 2) * S] = mul_mi(v[(2 + 4 * 2) * S]);                 // W^4 = -i
    v[(2 + 4 * 3) * S] = cmul(v[(2 + 4 * 3) * S], mk<T>(-h, -h));    // W^6
    v[(3 + 4 * 1) * S] = cmul(v[(3 + 4 * 1) * S], mk<T>(s1, -c1));   // W^3
    v[(3 + 4 * 2) * S] = cmul(v[(3 + 4 * 2) * S], mk<T>(-h, -h));    // W^6
    v[(3 + 4 * 3) * S] = cmul(v[(3 + 4 * 3) * S], mk<T>(-c1, s1));   // W^9
#pragma unroll
    for (int k2 = 0; k2 < 4; k2++) bfly4<T, S>(v + 4 * k2 * S);   // slot (k1 + 4 k2) holds X[k2 + 4 k1]
    // transpose the 4x4 slot grid so that slot k holds X[k]
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = a + 1; b < 4; b++) {
            cx<T> t = v[(a + 4 * b) * S];
            v[(a + 4 * b) * S] = v[(b + 4 * a) * S];
            v[(b + 4 * a) * S] = t;
        }
}

template <typename T, int S> __device__ __forceinline__ void bfly3(cx<T>* v)
{
    const T s = (T)0.86602540378443864676372317075294;  // sin(pi/3)
    cx<T> a = v[0], b = v[S], c = v[2 * S];
    cx<T> t = cadd(b, c), d = csub(b, c);
    cx<T> m = mk<T>(a.x - (T)0.5 * t.x, a.y - (T)0.5 * t.y);
    cx<T> r = mk<T>(s * d.y, -s * d.x);   // -i*s*d
    v[0] = cadd(a, t);
    v[S] = cadd(m, r);
    v[2 * S] = csub(m, r);
}

template <typename T, int S> __device__ __forceinline__ void bfly5(cx<T>* v)
{
    const T c1 = (T)0.30901699437494742410229341718282;   // cos(2pi/5)
    const T c2 = (T)-0.80901699437494742410229341718282;  // cos(4pi/5)
    const T s1 = (T)0.95105651629515357211643933337938;   // sin(2pi/5)
    const T s2 = (T)0.58778525229247312916870595463907;   // sin(4pi/5)
    cx<T> x0 = v[0];
    cx<T> p1 = cadd(v[S], v[4 * S]), m1 = csub(v[S], v[4 * S]);
    cx<T> p2 = cadd(v[2 * S], v[3 * S]), m2 = csub(v[2 * S], v[3 * S]);
    cx<T> a1 = mk<T>(x0.x + c1 * p1.x + c2 * p2.x, x0.y + c1 * p1.y + c2 * p2.y);
    cx<T> a2 = mk<T>(x0.x + c2 * p1.x + c1 * p2.x, x0.y + c2 * p1.y + c1 * p2.y);
    // -i * (s1 m1 + s2 m2), -i * (s2 m1 - s1 m2)
    cx<T> b1 = mk<T>(s1 * m1.y + s2 * m2.y, -(s1 * m1.x + s2 * m2.x));
    cx<T> b2 = mk<T>(s2 * m1.y - s1 * m2.y, -(s2 * m1.x - s1 * m2.x));
    v[0] = mk<T>(x0.x + p1.x + p2.x, x0.y + p1.y + p2.y);
    v[S] = cadd(a1, b1);
    v[4 * S] = csub(a1, b1);
    v[2 * S] = cadd(a2, b2);
    v[3 * S] = csub(a2, b2);
}

template <typename T, int S> __device__ __forceinline__ void bfly7(cx<T>* v)
{
    const T c1 = (T)0.62348980185873353052500488400424;
    const T c2 = (T)-0.22252093395631440428890256449679;
    const T c3 = (T)-0.90096886790241912623610231950745;
    const T s1 = (T)0.78183148246802980870844452667406;
    const T s2 = (T)0.97492791218182360701813168299393;
    const T s3 = (T)0.43388373911755812047576833284836;
    cx<T> x0 = v[0];
    cx<T> p1 = cadd(v[S], v[6 * S]), m1 = csub(v[S], v[6 * S]);
    cx<T> p2 = cadd(v[2 * S], v[5 * S]), m2 = csub(v[2 * S], v[5 * S]);
    cx<T> p3 = cadd(v[3 * S], v[4 * S]), m3 = csub(v[3 * S], v[4 * S]);
    cx<T> a1 = mk<T>(x0.x + c1 * p1.x + c2 * p2.x + c3 * p3.x, x0.y + c1 * p1.y + c2 * p2.y + c3 * p3.y);
    cx<T> a2 = mk<T>(x0.x + c2 * p1.x + c3 * p2.x + c1 * p3.x, x0.y + c2 * p1.y + c3 * p2.y + c1 * p3.y);
    cx<T> a3 = mk<T>(x0.x + c3 * p1.x + c1 * p2.x + c2 * p3.x, x0.y + c3 * p1.y + c1 * p2.y + c2 * p3.y);
    // X[k] = a_k - i * q_k, X[7-k] = a_k + i * q_k with q_k = sum_m sin(2 pi k m/7) m_m
    cx<T> q1 = mk<T>(s1 * m1.x + s2 * m2.x + s3 * m3.x, s1 * m1.y + s2 * m2.y + s3 * m3.y);
    cx<T> q2 = mk<T>(s2 * m1.x - s3 * m2.x - s1 * m3.x, s2 * m1.y - s3 * m2.y - s1 * m3.y);
    cx<T> q3 = mk<T>(s3 * m1.x - s1 * m2.x + s2 * m3.x, s3 * m1.y - s1 * m2.y + s2 * m3.y);
    cx<T> b1 = mul_mi(q1), b2 = mul_mi(q2), b3 = mul_mi(q3);
    v[0] = mk<T>(x0.x + p1.x + p2.x + p3.x, x0.y + p1.y + p2.y + p3.y);
    v[S] = cadd(a1, b1);
    v[6 * S] = csub(a1, b1);
    v[2 * S] = cadd(a2, b2);
    v[5 * S] = csub(a2, b2);
    v[3 * S] = cadd(a3, b3);
    v[4 * S] = csub(a3, b3);
}

template <int RAD, typename T, int S> __device__ __forceinline__ void bfly(cx<T>* v)
{
    if constexpr (RAD == 2) bfly2<T, S>(v);
    else if constexpr (RAD == 3) bfly3<T, S>(v);
    else if constexpr (RAD == 4) bfly4<T, S>(v);
    else if constexpr (RAD == 5) bfly5<T, S>(v);
    else if constexpr (RAD == 7) bfly7<T, S>(v);
    else if constexpr (RAD == 8) bfly8<T, S>(v);
    else if constexpr (RAD == 16) bfly16<T, S>(v);
    else static_assert(RAD == 2, "unsupported radix");
}

// ------------------------------------------------------------------------------------------
// Schedule: N points, R registers (points) per thread, radix list.  T = N/R threads cooperate on
// one line.  Thread t always holds positions t + u*T (u < R) of the line when it *reads*; the
// butterfly i (< R/RAD) of a stage works on registers u = i + m*(R/RAD) which are exactly the
// Stockham inputs j + m*N/RAD of butterfly j = t + i*T.  Outputs go to (j-k)*RAD + k + m*NS,
// k = j mod NS, through shared memory -- except in the last stage where that position is again
// t + u*T, i.e. the result is already in the right register for a coalesced store.
// ------------------------------------------------------------------------------------------
template <int N_, int R_, int... RADS> struct Sched {
    static constexpr int N = N_;
    static constexpr int R = R_;
    static constexpr int T = N_ / R_;
    static constexpr int NSTAGES = sizeof...(RADS);
    __host__ __device__ static constexpr int rad(int s)
    {
        const int r[sizeof...(RADS)] = {RADS...};
        return r[s];
    }
    __host__ __device__ static constexpr int ns(int s)
    {
        int p = 1;
        for (int i = 0; i < s; i++) p *= rad(i);
        return p;
    }
    // per-stage twiddle table: entries (m-1)*NS + k hold e^{-2 pi i k m / (NS*RAD)}, m = 1..RAD-1
    __host__ __device__ static constexpr int lut_off(int s)
    {
        int o = 0;
        for (int i = 1; i < s; i++) o += (rad(i) - 1) * ns(i);
        return o;
    }
    __host__ __device__ static constexpr int lut_size() { return lut_off(NSTAGES); }
    __host__ __device__ static constexpr bool valid()
    {
        int p = 1;
        for (int i = 0; i < NSTAGES; i++) {
            p *= rad(i);
            if (R_ % rad(i)) return false;
        }
        return p == N_ && N_ % R_ == 0;
    }
    // does butterfly i of stage s use the same k for every i?  (then one twiddle set per stage)
    __host__ __device__ static constexpr bool shared_k(int s) { return ns(s) <= T && T % ns(s) == 0; }
    __host__ __device__ static constexpr int tw_regs(int s) { return s == 0 ? 0 : (shared_k(s) ? 1 : R_ / rad(s)) * (rad(s) - 1); }
    __host__ __device__ static constexpr int tw_regs_total()
    {
        int o = 0;
        for (int i = 1; i < NSTAGES; i++) o += tw_regs(i);
        return o;
    }
};

// shared-memory line layout: one padding element every 2^PS elements, so that the stride-RAD
// writes of the first exchange and the stride-1 reads land in distinct 16-byte bank groups.
template <typename T> struct SmemGeom {
    // W = complex elements per 128-byte shared-memory wavefront (8 for double2, 16 for float2)
    static constexpr int W = 128 / (2 * sizeof(T));
    static constexpr int PS = sizeof(T) == 8 ? 3 : 4;
    __host__ __device__ static constexpr int pad(int e) { return e + (e >> PS); }
    // Line pitch for C lines per tile.  In the column-fastest thread map a wavefront covers
    // min(C, W) columns x W/C consecutive butterflies whose padded positions are consecutive
    // (mod W), so the pitch must be = W/C (mod W) for the W lanes to fall in W distinct banks;
    // the line-fastest map is conflict free for any pitch.
    __host__ __device__ static constexpr int line(int n, int C)
    {
        int want = C >= W ? 1 : W / C;
        int l = n + (n >> PS);
        while (l % W != want % W) l++;
        return l;
    }
};

// twiddle application + butterflies of stage s on registers v[R]
template <class S, int s, typename T, bool TWREG>
__device__ __forceinline__ void stage_compute(cx<T>* v, int t, const cx<T>* __restrict__ lut, const cx<T>* twr)
{
    constexpr int RAD = S::rad(s), NS = S::ns(s), NB = S::R / RAD;
    if constexpr (s > 0) {
        constexpr int off = S::lut_off(s);
        constexpr bool shared = S::shared_k(s);
#pragma unroll
        for (int i = 0; i < NB; i++) {
            const int k = (t + i * S::T) % NS;
#pragma unroll
            for (int m = 1; m < RAD; m++) {
                cx<T> w;
                if constexpr (TWREG) w = twr[(shared ? 0 : i * (RAD - 1)) + (m - 1)];
                else w = lut[off + (m - 1) * NS + k];
                v[i + m * NB] = cmul(v[i + m * NB], w);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < NB; i++) bfly<RAD, T, NB>(v + i);
}

// load this thread's twiddles of stage s into registers (twr must have S::tw_regs(s) entries)
template <class S, int s, typename T>
__device__ __forceinline__ void stage_load_tw(cx<T>* twr, int t, const cx<T>* __restrict__ lut)
{
    constexpr int RAD = S::rad(s), NS = S::ns(s), NB = S::R / RAD;
    constexpr int off = S::lut_off(s);
    constexpr bool shared = S::shared_k(s);
#pragma unroll
    for (int i = 0; i < (shared ? 1 : NB); i++) {
        const int k = (t + i * S::T) % NS;
#pragma unroll
        for (int m = 1; m < RAD; m++) twr[i * (RAD - 1) + (m - 1)] = lut[off + (m - 1) * NS + k];
    }
}

// write the outputs of stage s (thread-in-line index t) into a padded smem line
template <class S, int s, typename T>
__device__ __forceinline__ void stage_scatter(const cx<T>* v, int t, cx<T>* line)
{
    constexpr int RAD = S::rad(s), NS = S::ns(s), NB = S::R / RAD;
#pragma unroll
    for (int i = 0; i < NB; i++) {
        const int j = t + i * S::T;
        const int k = j % NS;
        const int j0 = (j - k) * RAD + k;
#pragma unroll
        for (int m = 0; m < RAD; m++) line[SmemGeom<T>::pad(j0 + m * NS)] = v[i + m * NB];
    }
}

// read positions t + u*T of a padded smem line
template <class S, typename T>
__device__ __forceinline__ void stage_gather(cx<T>* v, int t, const cx<T>* line)
{
#pragma unroll
    for (int u = 0; u < S::R; u++) v[u] = line[SmemGeom<T>::pad(t + u * S::T)];
}

// ------------------------------------------------------------------------------------------
// TMA bulk copy (cp.async.bulk, SASS UBLKCP) used to stage the twiddle tile into shared memory
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t phase)
{
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase) : "memory");
    return ok != 0;
}
// One timeout policy for every device-side wait (mbarrier, in-device plane counters, cross-device arrival flags): a wait
// that has not been satisfied after DFFT_SPIN_TIMEOUT_NS of wall-clock time (%globaltimer) is a lost dependency -- a peer
// that died, a transaction that can never complete -- and traps, so the host sees a launch failure instead of a GPU that
// hangs forever.  The bound is far above any legitimate skew (process start-up, lazy module load, a peer's own waits).
constexpr unsigned long long DFFT_SPIN_TIMEOUT_NS = 120ull * 1000ull * 1000ull * 1000ull;
__device__ __forceinline__ unsigned long long gtime_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
struct SpinGuard {
    unsigned long long t0 = 0;
    unsigned n = 0;
    __device__ __forceinline__ void tick()
    {
        if ((++n & 1023u) == 0) {
            const unsigned long long now = gtime_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > DFFT_SPIN_TIMEOUT_NS) __trap();
        }
    }
};
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase)
{
    SpinGuard g;
    while (!mbar_try_wait(bar, phase)) g.tick();
}
__device__ __forceinline__ void fence_barrier_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// global -> shared bulk copy of `bytes` (multiple of 16, both 16-byte aligned), completes on bar
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// Stage the per-length twiddle table (global, built at plan time) into shared memory with one
// TMA bulk copy issued by thread 0; everyone waits on the mbarrier.  `bar` and `dst` in smem.
// The global table is allocated padded to a multiple of 16 bytes (build_lut), `dst` is 16-byte aligned.
template <typename T>
__device__ __forceinline__ void stage_twiddles_tma(cx<T>* dst, const cx<T>* __restrict__ src, int entries, uint64_t* bar)
{
    if (entries == 0) return;
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t bytes = (uint32_t)((entries * sizeof(cx<T>) + 15) / 16 * 16);
        mbar_expect_tx(bar, bytes);
        tma_bulk_g2s(dst, src, bytes, bar);
    }
    mbar_wait(bar, 0);
}

}  // namespace dfft
