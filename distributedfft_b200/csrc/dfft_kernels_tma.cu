// dfft_kernels_tma.cu -- instantiations and host-side helpers of the TMA-pipelined pass kernels (fft_tma.cuh).
#include <cuda.h>

#include <mutex>

#include "dfft_kernels.cuh"
#include "dfft_launch.cuh"
#include "fft_tma.cuh"

namespace dfft {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
        cudaGetLastError();
    });
    return fn;
}

bool tma_available() { return encode_fn() != nullptr; }

// 3-D tensor of complex elements: dim0 (fastest, contiguous) d0, dim1 d1 with stride s1, dim2 d2 with stride s2 (strides in complex
// elements); box (b0, b1, b2).  `map` points to 128 bytes, 64-byte aligned (a CUtensorMap).
// L2 promotion: 256 B, except for 128-byte box rows, which are promoted to one row.  Measured on H100 (DESIGN.md 3.4): at
// 512^3 fp64 (C = 8, 128-byte rows) 256 B took the fused t0 2.08 against 2.05-2.06 ms and the TMA_XF pass 1.61 against
// 1.58 ms, and 512^3 fp32 (C = 16) was a tie.  Narrower rows (64 B) were not measured apart from run-to-run noise, so they
// keep 256 B
int tma_encode_3d(void* map, void* base, int prec, long long d0, long long d1, long long d2, long long s1, long long s2, int b0, int b1, int b2)
{
    EncodeTiledFn fn = encode_fn();
    if (!fn) return -1;
    const size_t esz = prec == 0 ? 16 : 8;
    cuuint64_t dims[3] = {(cuuint64_t)d0 * 2, (cuuint64_t)d1, (cuuint64_t)d2};
    cuuint64_t strides[2] = {(cuuint64_t)s1 * esz, (cuuint64_t)s2 * esz};
    cuuint32_t box[3] = {(cuuint32_t)b0 * 2, (cuuint32_t)b1, (cuuint32_t)b2};
    cuuint32_t estr[3] = {1, 1, 1};
    const CUtensorMapL2promotion promo = (size_t)b0 * esz == 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
    const CUresult r = fn((CUtensorMap*)map, prec == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT64 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, base, dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

// The TMA kernels run one CTA per SM (their rings fill its shared memory), so they need the shared-memory opt-in but no
// occupancy query
template <class S, typename T, int C, int M>
static cudaError_t launch_tma_mode(const TmaArgs<T>& a, const CUtensorMap& mi, const CUtensorMap& mo, int sm_count, cudaStream_t st)
{
    constexpr auto kern = fft_tma_pass_kernel<S, T, C, M>;
    constexpr size_t smem = TmaGeom<S, T, C>::PASS_SMEM;
    const cudaError_t e = smem_optin<kern>(smem);
    if (e != cudaSuccess || a.ntiles <= 0) return e;
    kern<<<(unsigned)grid_for(sm_count, 1, 0, a.ntiles), S::T * C, smem, st>>>(a, mi, mo);
    return cudaGetLastError();
}

template <class S, typename T, int C>
static cudaError_t launch_tma(int mode, const void* vargs, const void* map_in, const void* map_out, int sm_count, cudaStream_t st)
{
    const TmaArgs<T>& a = *reinterpret_cast<const TmaArgs<T>*>(vargs);
    static CUtensorMap dummy{};
    const CUtensorMap& mi = map_in ? *reinterpret_cast<const CUtensorMap*>(map_in) : dummy;
    const CUtensorMap& mo = map_out ? *reinterpret_cast<const CUtensorMap*>(map_out) : dummy;
    switch (mode) {
        case TMA_Z: return launch_tma_mode<S, T, C, TMA_Z>(a, mi, mo, sm_count, st);
        case TMA_Y: return launch_tma_mode<S, T, C, TMA_Y>(a, mi, mo, sm_count, st);
        case TMA_XF: return launch_tma_mode<S, T, C, TMA_XF>(a, mi, mo, sm_count, st);
        case TMA_XB: return launch_tma_mode<S, T, C, TMA_XB>(a, mi, mo, sm_count, st);
        default: return cudaErrorInvalidValue;
    }
}

template <class S, typename T, int C>
static cudaError_t launch_tma_fused_zy(const void* vargs, const FusedCtl* ctl, const void* map_mid, int sm_count, cudaStream_t st)
{
    const TmaFusedArgs<T>& a = *reinterpret_cast<const TmaFusedArgs<T>*>(vargs);
    using G_ = TmaGeom<S, T, C>;
    constexpr auto kern = fft_tma_fused_zy_kernel<S, T, C>;
    const cudaError_t e = smem_optin<kern>(G_::SMEM);
    if (e != cudaSuccess) return e;
    if (ctl->planes <= 0) return cudaSuccess;
    const long long total = ctl->planes * ((long long)ctl->GA + ctl->GB);
    if (total >= (1ll << 31)) return cudaErrorInvalidConfiguration;   // the kernel decodes tickets in 32 bits
    const long long grid = grid_for(sm_count, 1, 0, total);
    FusedCtl c = *ctl;
    // the Z role runs ahead of the Y role by the tiles the rings hold beside the ones each CTA is transforming
    // (NSLOT - NGROUP per CTA): 3 planes at 512 points on 132 SMs.  Each plane more keeps another 4 MiB of intermediate in
    // the L2; on tma_ring at 512^3 fp64 on H100, lag 2 measured 0.15 ms and lag 4 0.03 ms slower than lag 3 (DESIGN.md 3.4)
    if (c.lag <= 0) c.lag = (int)((grid * (G_::NSLOT - G_::NGROUP) + c.GA + c.GB - 1) / ((long long)c.GA + c.GB));
    kern<<<(unsigned)grid, TMA_CONSUMERS + 32, G_::SMEM, st>>>(a, c, *reinterpret_cast<const CUtensorMap*>(map_mid));
    return cudaGetLastError();
}

template <class S, typename T, int C, bool FUSED_ZY = false> static TmaEntry make_tma_entry(unsigned use)
{
    TmaEntry e{};
    e.use = use;
    e.N = S::N;
    e.prec = sizeof(T) == 8 ? 0 : 1;
    e.C = C;
    e.rows = TmaGeom<S, T, C>::ROWS;
    e.nstages = S::NSTAGES;
    for (int i = 0; i < S::NSTAGES; i++) e.rad[i] = S::rad(i);
    e.launch = launch_tma<S, T, C>;
    if constexpr (FUSED_ZY) e.fused_zy = launch_tma_fused_zy<S, T, C>;
    return e;
}

// per length: the default entry, and its copy with every pass mode switched on (DFFT_TMA=2).  A plan keeps pointers to the
// entries of its three axes, so both tables are built once and never change
struct TmaTables { std::vector<TmaEntry> dflt, forced; };
static const TmaTables& tma_tables()
{
    static TmaTables tt;
    static std::once_flag once;
    std::call_once(once, [] {
        std::vector<TmaEntry>& t = tt.dflt;
        // tile = C lines of N points = 64 KB (48 KB for 768), S::T * C threads, one CTA per SM
        // which modes to use: per pass, whichever of the TMA and the register-staged kernel was faster at N^3 on one GPU
        // (chosen on an earlier GPU generation; 512 fp64 re-checked on H100, DESIGN.md section 7)
        constexpr unsigned Z = 1u << TMA_Z, Y = 1u << TMA_Y, XF = 1u << TMA_XF, X = XF | (1u << TMA_XB), ZY = 1u << TMA_USE_ZY;
        // H100: forward X faster, Z a tie; X backward not measured; the fused forward t0 beats the Z + Y sweeps (DESIGN.md 3.4)
        t.push_back(make_tma_entry<Sched<512, 8, 8, 8, 8>, double, 8, true>(Y | XF | ZY));
        t.push_back(make_tma_entry<Sched<1024, 8, 8, 8, 8, 2>, double, 4>(Y | X));
        t.push_back(make_tma_entry<Sched<256, 8, 8, 8, 4>, double, 16>(Z | Y | X));
        t.push_back(make_tma_entry<Sched<768, 12, 4, 4, 4, 4, 3>, double, 4>(Y));
        t.push_back(make_tma_entry<Sched<512, 16, 8, 8, 8>, float, 16>(Z | Y | X));
        t.push_back(make_tma_entry<Sched<1024, 16, 16, 8, 8>, float, 8>(Y | X));
        t.push_back(make_tma_entry<Sched<768, 12, 4, 4, 4, 4, 3>, float, 8>(Y | X));
        // the forced copies keep bit TMA_USE_ZY: the fused forward t0 stays the default where it is one
        tt.forced = t;
        for (TmaEntry& e : tt.forced) e.use |= Z | Y | X;
    });
    return tt;
}

const TmaEntry* find_tma_entry(int N, int prec)
{
    const char* env = getenv("DFFT_TMA");
    if (env && atoi(env) == 0) return nullptr;
    if (getenv("DFFT_GENERIC") && atoi(getenv("DFFT_GENERIC")) != 0) return nullptr;
    if (!tma_available()) return nullptr;
    const TmaTables& tt = tma_tables();
    const std::vector<TmaEntry>& t = env && atoi(env) == 2 ? tt.forced : tt.dflt;
    for (const TmaEntry& e : t)
        if (e.N == N && e.prec == prec) return &e;
    return nullptr;
}

}  // namespace dfft
