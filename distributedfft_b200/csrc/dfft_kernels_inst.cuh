// dfft_kernels_inst.cuh -- launcher template + size-table macros, included by the per-precision
// instantiation units.
#pragma once
#include <type_traits>
#include "dfft_kernels.cuh"
#include "dfft_launch.cuh"

namespace dfft {

// Every launcher below picks its kernel, block size, dynamic shared memory and argument struct, and sizes its persistent grid
// with resident_grid (dfft_launch.cuh).  Only launch_pass (and launch_generic) cap the resident CTAs per SM with
// TileArgs::max_ctas_per_sm: the pipelined Y and X passes are the only passes that set it
template <class S, typename T, int C, int MI, int MO, bool TW, bool CI, bool CO, int MINB, bool PP, bool EPI = false>
cudaError_t launch_pass(const void* vargs, int sm_count, cudaStream_t st)
{
    const TileArgs<T>& a = *reinterpret_cast<const TileArgs<T>*>(vargs);
    constexpr auto kern = fft_tile_kernel<S, T, C, MI, MO, TW, CI, CO, MINB, PP, false, EPI>;
    constexpr size_t smem = TileSmem<S, T, C, PP>::bytes(CI || CO);
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(S::T * C, smem, a.max_ctas_per_sm, a.ntiles, sm_count, grid);
    if (e != cudaSuccess || grid == 0) return e;
    kern<<<(unsigned)grid, S::T * C, smem, st>>>(a);
    return cudaGetLastError();
}

// real-data Z passes (fft_real.cuh): vargs is a RealZArgs<T>
template <class S, typename T, int C, bool TW, int MINB, bool PP, bool C2R>
cudaError_t launch_real(const void* vargs, int sm_count, cudaStream_t st)
{
    const RealZArgs<T>& a = *reinterpret_cast<const RealZArgs<T>*>(vargs);
    constexpr auto kern = [] {   // only the kernel of this direction is instantiated
        if constexpr (C2R) return fft_z_c2r_kernel<S, T, C, TW, MINB, PP>;
        else return fft_z_r2c_kernel<S, T, C, TW, MINB, PP>;
    }();
    constexpr size_t smem = TileSmem<S, T, C, PP>::bytes(false);
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(S::T * C, smem, 0, a.t.ntiles, sm_count, grid);
    if (e != cudaSuccess || grid == 0) return e;
    kern<<<(unsigned)grid, S::T * C, smem, st>>>(a);
    return cudaGetLastError();
}

// spectral convolution column pass (fft_conv_kernel, or fft_conv_shared_kernel when ConvArgs::mult_shared): vargs is a ConvArgs<T>
template <class S, typename T, int C, bool TW, bool CO, int MINB, bool PP, bool SH>
cudaError_t launch_conv_k(const ConvArgs<T>& a, int sm_count, cudaStream_t st)
{
    constexpr auto kern = [] {   // only the kernel of this mode is instantiated
        if constexpr (SH) return fft_conv_shared_kernel<S, T, C, TW, MINB, PP>;
        else return fft_conv_kernel<S, T, C, TW, CO, MINB, PP>;
    }();
    constexpr size_t smem = TileSmem<S, T, C, PP>::bytes(CO);
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(S::T * C, smem, 0, a.t.ntiles, sm_count, grid);
    if (e != cudaSuccess || grid == 0) return e;
    kern<<<(unsigned)grid, S::T * C, smem, st>>>(a);
    return cudaGetLastError();
}

template <class S, typename T, int C, bool TW, bool CO, int MINB, bool PP>
cudaError_t launch_conv(const void* vargs, int sm_count, cudaStream_t st)
{
    const ConvArgs<T>& a = *reinterpret_cast<const ConvArgs<T>*>(vargs);
    if constexpr (!CO) {   // the shared multiplier exists for the local-store kind only
        if (a.mult_shared) return launch_conv_k<S, T, C, TW, CO, MINB, PP, true>(a, sm_count, st);
    } else {
        if (a.mult_shared) return cudaErrorInvalidValue;
    }
    return launch_conv_k<S, T, C, TW, CO, MINB, PP, false>(a, sm_count, st);
}

// 1-D convolution of contiguous lines (fft_line_conv_kernel: vargs is a LineConvArgs<T>; R2C: fft_line_conv_r2c_kernel, vargs is
// a RealLineConvArgs<T>)
template <class S, typename T, int C, bool TW, int MINB, bool PP, bool R2C>
cudaError_t launch_line_conv(const void* vargs, int sm_count, cudaStream_t st)
{
    using Args = std::conditional_t<R2C, RealLineConvArgs<T>, LineConvArgs<T>>;
    const Args& a = *reinterpret_cast<const Args*>(vargs);
    constexpr auto kern = [] {   // only the kernel of this kind is instantiated
        if constexpr (R2C) return fft_line_conv_r2c_kernel<S, T, C, TW, MINB, PP>;
        else return fft_line_conv_kernel<S, T, C, TW, MINB, PP>;
    }();
    constexpr size_t smem = TileSmem<S, T, C, PP>::bytes(false);
    const TileArgs<T>& t = [&]() -> const TileArgs<T>& { if constexpr (R2C) return a.r.t; else return a.t; }();
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(S::T * C, smem, 0, t.ntiles, sm_count, grid);
    if (e != cudaSuccess || grid == 0) return e;
    kern<<<(unsigned)grid, S::T * C, smem, st>>>(a);
    return cudaGetLastError();
}

// the zero-padded 1-D convolve lines plans' kinds: vargs is a PadArgs<T>; PK_LINE_CONV_PAD runs fft_line_conv_pad_kernel,
// PK_XF_TW_PAD / PK_XB_TW_PAD the forward / inverse fft_four_step_pad_kernel
template <class S, typename T, int C, bool TW, int MINB, bool PP, int KIND>
cudaError_t launch_pad(const void* vargs, int sm_count, cudaStream_t st)
{
    const PadArgs<T>& a = *reinterpret_cast<const PadArgs<T>*>(vargs);
    constexpr auto kern = [] {   // only the kernel of this kind is instantiated
        if constexpr (KIND == PK_LINE_CONV_PAD) return fft_line_conv_pad_kernel<S, T, C, TW, MINB, PP>;
        else return fft_four_step_pad_kernel<S, T, C, TW, MINB, PP, KIND == PK_XF_TW_PAD>;
    }();
    constexpr size_t smem = TileSmem<S, T, C, PP>::bytes(false);
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(S::T * C, smem, 0, a.c.t.ntiles, sm_count, grid);
    if (e != cudaSuccess || grid == 0) return e;
    kern<<<(unsigned)grid, S::T * C, smem, st>>>(a);
    return cudaGetLastError();
}

// the real zero-padded 1-D convolve lines plans' kinds: vargs is a RealPadArgs<T>; PK_LINE_CONV_PAD_R2C runs
// fft_line_conv_pad_r2c_kernel, PK_XF_TW_PAD_R2C / PK_XB_TW_PAD_C2R the real fft_four_step_pad_kernel, PK_XCONV_R2C fft_conv_r2c_kernel
template <class S, typename T, int C, bool TW, int MINB, bool PP, int KIND>
cudaError_t launch_real_pad(const void* vargs, int sm_count, cudaStream_t st)
{
    const RealPadArgs<T>& a = *reinterpret_cast<const RealPadArgs<T>*>(vargs);
    constexpr auto kern = [] {   // only the kernel of this kind is instantiated
        if constexpr (KIND == PK_LINE_CONV_PAD_R2C) return fft_line_conv_pad_r2c_kernel<S, T, C, TW, MINB, PP>;
        else if constexpr (KIND == PK_XCONV_R2C) return fft_conv_r2c_kernel<S, T, C, TW, MINB, PP>;
        else return fft_four_step_pad_kernel<S, T, C, TW, MINB, PP, KIND == PK_XF_TW_PAD_R2C, true>;
    }();
    constexpr size_t smem = TileSmem<S, T, C, PP>::bytes(false);
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(S::T * C, smem, 0, a.c.r.t.ntiles, sm_count, grid);
    if (e != cudaSuccess || grid == 0) return e;
    kern<<<(unsigned)grid, S::T * C, smem, st>>>(a);
    return cudaGetLastError();
}

// X + Y passes of square planes (fft_plane_kernel): vargs is a PlaneArgs<T>; P planes per CTA
template <class S, typename T, int P, int MINB>
cudaError_t launch_plane(const void* vargs, int sm_count, cudaStream_t st)
{
    const PlaneArgs<T>& a = *reinterpret_cast<const PlaneArgs<T>*>(vargs);
    constexpr auto kern = fft_plane_kernel<S, T, P, MINB>;
    constexpr size_t smem = PlaneSmem<S, T, P>::bytes;
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(S::T * S::N * P, smem, 0, (a.planes + P - 1) / P, sm_count, grid);
    if (e != cudaSuccess || grid == 0) return e;
    kern<<<(unsigned)grid, S::T * S::N * P, smem, st>>>(a);
    return cudaGetLastError();
}

// 2-D convolution of whole square images (fft_plane_conv_kernel): vargs is a PlaneConvArgs<T>; P images per CTA
template <class S, typename T, int P, int MINB>
cudaError_t launch_plane_conv(const void* vargs, int sm_count, cudaStream_t st)
{
    const PlaneConvArgs<T>& a = *reinterpret_cast<const PlaneConvArgs<T>*>(vargs);
    constexpr auto kern = fft_plane_conv_kernel<S, T, P, MINB>;
    constexpr size_t smem = PlaneSmem<S, T, P>::bytes;
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(S::T * S::N * P, smem, 0, (a.p.planes + P - 1) / P, sm_count, grid);
    if (e != cudaSuccess || grid == 0) return e;
    kern<<<(unsigned)grid, S::T * S::N * P, smem, st>>>(a);
    return cudaGetLastError();
}

// Dynamic shared memory of the multi-role kernels: one exchange buffer (the largest role's) + every role's own twiddles, barrier
// and chunk tables.  sm_90 grants at most 227 KB per block; a combination above that cannot be launched, so its entry is left
// null and plans run the separate passes instead (4096 fp64: two 64 KB twiddle tables + a 136 KB exchange buffer; 2048 fp64 with
// the chunk tables of the peer-store / unpack roles)
constexpr size_t SMEM_OPTIN_MAX = 227 * 1024;
template <class... Ops> constexpr size_t roles_smem()
{
    size_t exch = 0;
    ((exch = Ops::SM::exch_bytes > exch ? Ops::SM::exch_bytes : exch), ...);
    return exch + (Ops::aux_bytes + ...);
}

// The multi-role kernels below decode their tickets in 32 bits: a launch of 2^31 or more tickets is refused
template <class OpA, class OpB, typename T, int MINB>
cudaError_t launch_fused(const void* va, const void* vb, const FusedCtl* ctl, int sm_count, cudaStream_t st)
{
    const TileArgs<T>& a = *reinterpret_cast<const TileArgs<T>*>(va);
    const TileArgs<T>& b = *reinterpret_cast<const TileArgs<T>*>(vb);
    constexpr auto kern = fft_fused2_kernel<OpA, OpB, T, MINB>;
    constexpr size_t smem = roles_smem<OpA, OpB>();
    const long long total = ctl->planes > 0 ? ctl->planes * ((long long)ctl->GA + ctl->GB) : 0;
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(OpA::NT, smem, 0, total, sm_count, grid);
    if (e != cudaSuccess) return e;
    if (total >= (1ll << 31)) return cudaErrorInvalidConfiguration;
    if (grid == 0) return cudaSuccess;
    FusedCtl c = *ctl;
    if (c.lag <= 0) c.lag = (int)((grid + c.GA + c.GB - 1) / ((long long)c.GA + c.GB)) + 1;   // role A stays one in-flight window ahead
    kern<<<(unsigned)grid, OpA::NT, smem, st>>>(a, b, c);
    return cudaGetLastError();
}

template <class OpA, class OpB, typename T, int MINB>
cudaError_t launch_fused_yx(const void* va, const void* vb, const YxCtl* ctl, int sm_count, cudaStream_t st)
{
    const TileArgs<T>& a = *reinterpret_cast<const TileArgs<T>*>(va);
    const TileArgs<T>& b = *reinterpret_cast<const TileArgs<T>*>(vb);
    constexpr auto kern = fft_fused_yx_kernel<OpA, OpB, T, MINB>;
    constexpr size_t smem = roles_smem<OpA, OpB>();
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(OpA::NT, smem, 0, (long long)ctl->TA + ctl->TB, sm_count, grid);
    if (e != cudaSuccess || grid == 0) return e;
    kern<<<(unsigned)grid, OpA::NT, smem, st>>>(a, b, *ctl);
    return cudaGetLastError();
}

template <class OpA, class OpB, class OpC, typename T, int MINB>
cudaError_t launch_fused3(const void* va, const void* vb, const void* vc, const Fused3Ctl* ctl, int sm_count, cudaStream_t st)
{
    const TileArgs<T>& a = *reinterpret_cast<const TileArgs<T>*>(va);
    const TileArgs<T>& b = *reinterpret_cast<const TileArgs<T>*>(vb);
    const TileArgs<T>& c = *reinterpret_cast<const TileArgs<T>*>(vc);
    constexpr auto kern = fft_fused3_kernel<OpA, OpB, OpC, T, MINB>;
    constexpr size_t smem = roles_smem<OpA, OpB, OpC>();
    const long long total = ctl->planes > 0 ? ctl->planes * ((long long)ctl->GA + ctl->GB) + ctl->rows * (long long)ctl->GX : 0;
    long long grid = 0;
    const cudaError_t e = resident_grid<kern>(OpA::NT, smem, 0, total, sm_count, grid);
    if (e != cudaSuccess) return e;
    if (total >= (1ll << 31)) return cudaErrorInvalidConfiguration;
    if (grid == 0) return cudaSuccess;
    Fused3Ctl f = *ctl;
    if (f.lag <= 0) f.lag = (int)((grid + f.GA + f.GBk - 1) / ((long long)f.GA + f.GBk)) + 1;
    kern<<<(unsigned)grid, OpA::NT, smem, st>>>(a, b, c, f);
    return cudaGetLastError();
}

template <class OpA, class OpB, typename T, int MINB> constexpr FusedLaunchFn fused_if_fits()
{
    if constexpr (roles_smem<OpA, OpB>() <= SMEM_OPTIN_MAX) return launch_fused<OpA, OpB, T, MINB>;
    else return nullptr;
}

// lines per tile of a configuration whose load or store goes through the chunk tables: C, halved until the tile's exchange
// buffer, its twiddles and the chunk tables fit in one block's shared memory (4096-point fp64: 2 -> 1; every other tuned
// configuration keeps its C)
template <class S, typename T, int C, bool PP> constexpr int chunked_C()
{
    if constexpr (C > 1 && TileSmem<S, T, C, PP>::bytes(true) > SMEM_OPTIN_MAX) return chunked_C<S, T, C / 2, PP>();
    else return C;
}

template <class S> void fill_rad(int& n, int* rad)
{
    n = S::NSTAGES;
    for (int i = 0; i < S::NSTAGES; i++) rad[i] = S::rad(i);
}

// One kernel configuration: schedule, lines per tile, twiddles in registers, min CTAs/SM, ping-pong exchange buffer
template <class S_, int C_, bool TW_, int MB_, bool PP_> struct Cfg {
    using S = S_;
    static constexpr int C = C_, MB = MB_;
    static constexpr bool TW = TW_, PP = PP_;
};

// Z: contiguous pass.  Y: strided pass on local memory (t0 axis-1, backward unpack).  X: the t3 passes (strided on one
// side, contiguous on the other).  PEER: the Y pass with the chunked store (pack / peer receive buffers over NVLink),
// which wants >= 128-byte row segments; must use Y's schedule (it shares the twiddle table).
// FH bit 0: the fused t0 kernels carry L2 eviction hints (first role: streamed input evict_first, intermediate evict_last;
// second role: intermediate and output evict_first); FH bit 1: the contiguous role of the fused kernels synchronises per
// line (named barriers) instead of per CTA -- experiments, see DESIGN.md
template <class G, int C_> using WithC = Cfg<typename G::S, C_, G::TW, G::MB, G::PP>;

template <typename T, class Z, class Y, class X = Y, class PEER_ = Y, int FH = 0>
SizeEntry make_entry(int variant = 0)
{
    using ZS = typename Z::S;
    using SS = typename Y::S;
    using XS = typename X::S;
    static_assert(std::is_same<typename PEER_::S, SS>::value, "the peer-store configuration shares the Y schedule");
    // the chunked kinds in configurations that can be launched (chunked_C)
    using PEER = WithC<PEER_, chunked_C<SS, T, PEER_::C, PEER_::PP>()>;
    using YCI = WithC<Y, chunked_C<SS, T, Y::C, Y::PP>()>;
    using XCO = WithC<X, chunked_C<XS, T, X::C, X::PP>()>;
    SizeEntry e{};
    e.N = ZS::N;
    e.variant = variant;
    e.prec = sizeof(T) == 8 ? 0 : 1;
    e.z_C = Z::C;
    e.s_C = Y::C;
    e.p_C = PEER::C;
    e.x_C = X::C;
    e.ci_C = YCI::C;
    e.xo_C = XCO::C;
    fill_rad<ZS>(e.z_nstages, e.z_rad);
    fill_rad<SS>(e.s_nstages, e.s_rad);
    fill_rad<XS>(e.x_nstages, e.x_rad);
    e.launch[PK_Z] = launch_pass<ZS, T, Z::C, MAP_T, MAP_T, Z::TW, false, false, Z::MB, Z::PP>;
    e.launch[PK_Y] = launch_pass<SS, T, Y::C, MAP_C, MAP_C, Y::TW, false, false, Y::MB, Y::PP>;
    e.launch[PK_Y_CO] = launch_pass<SS, T, PEER::C, MAP_C, MAP_C, PEER::TW, false, true, PEER::MB, PEER::PP>;
    e.launch[PK_Y_CI] = launch_pass<SS, T, YCI::C, MAP_C, MAP_C, YCI::TW, true, false, YCI::MB, YCI::PP>;
    e.launch[PK_XF] = launch_pass<XS, T, X::C, MAP_C, MAP_T, X::TW, false, false, X::MB, X::PP>;
    e.launch[PK_XB] = launch_pass<XS, T, X::C, MAP_T, MAP_C, X::TW, false, false, X::MB, X::PP>;
    e.launch[PK_XB_CO] = launch_pass<XS, T, XCO::C, MAP_T, MAP_C, XCO::TW, false, true, XCO::MB, XCO::PP>;
    e.launch[PK_XF_TW] = launch_pass<XS, T, X::C, MAP_C, MAP_T, X::TW, false, false, X::MB, X::PP, true>;
    // real-data Z passes with the contiguous configuration (C line pairs per tile); default entries only -- the alternate
    // tunings are experiments on the C2C path.  Twiddles come from shared memory (TWREG off): the pair loads and the split
    // epilogue need the registers the twiddles would hold, and register twiddles spilled at 512 / 1024.  The inverse loads two
    // lines per point and runs with one resident CTA less than the forward (no spills at 1024 fp32 otherwise)
    if (variant == 0) {
        constexpr int MBI = Z::MB > 3 ? 3 : Z::MB;
        e.launch[PK_Z_R2C] = launch_real<ZS, T, Z::C, false, Z::MB, Z::PP, false>;
        e.launch[PK_Z_C2R] = launch_real<ZS, T, Z::C, false, MBI, Z::PP, true>;
        // spectral convolution along x (the X axis of a convolve plan uses this entry's strided schedule and twiddle table)
        e.launch[PK_XCONV] = launch_conv<SS, T, Y::C, Y::TW, false, Y::MB, Y::PP>;
        e.launch[PK_XCONV_CO] = launch_conv<SS, T, PEER::C, PEER::TW, true, PEER::MB, PEER::PP>;
        // 1-D convolution of contiguous lines in the contiguous configuration: the complex kernel with the Z pass's register
        // budget, the real one with the real kernels' (shared-memory twiddles, MBI)
        e.launch[PK_LINE_CONV] = launch_line_conv<ZS, T, Z::C, Z::TW, Z::MB, Z::PP, false>;
        e.launch[PK_LINE_CONV_R2C] = launch_line_conv<ZS, T, Z::C, false, MBI, Z::PP, true>;
        // the zero-padded 1-D convolution: the short path in PK_LINE_CONV's configuration, the long path's outer passes in the X
        // configuration of PK_XF_TW and PK_XB
        e.launch[PK_LINE_CONV_PAD] = launch_pad<ZS, T, Z::C, Z::TW, Z::MB, Z::PP, PK_LINE_CONV_PAD>;
        e.launch[PK_XF_TW_PAD] = launch_pad<XS, T, X::C, X::TW, X::MB, X::PP, PK_XF_TW_PAD>;
        e.launch[PK_XB_TW_PAD] = launch_pad<XS, T, X::C, X::TW, X::MB, X::PP, PK_XB_TW_PAD>;
        // the real zero-padded 1-D convolution: the short path in PK_LINE_CONV_R2C's configuration, the long path's outer passes in
        // the X configuration, its middle pass in PK_XCONV's
        e.launch[PK_LINE_CONV_PAD_R2C] = launch_real_pad<ZS, T, Z::C, false, MBI, Z::PP, PK_LINE_CONV_PAD_R2C>;
        e.launch[PK_XF_TW_PAD_R2C] = launch_real_pad<XS, T, X::C, X::TW, X::MB, X::PP, PK_XF_TW_PAD_R2C>;
        e.launch[PK_XCONV_R2C] = launch_real_pad<SS, T, Y::C, Y::TW, Y::MB, Y::PP, PK_XCONV_R2C>;
        e.launch[PK_XB_TW_PAD_C2R] = launch_real_pad<XS, T, X::C, X::TW, X::MB, X::PP, PK_XB_TW_PAD_C2R>;
        // X and Y passes of whole square planes in one kernel, where both roles share one schedule (and so one twiddle table).
        // Register budget: 64 per thread (2 CTAs of 512 / 4 of 256 threads), except 32-point fp64, which spills at 64 and is
        // given 85 (3 CTAs of 256); 64-point fp64 keeps 2 CTAs of 512 with a small spill (DESIGN.md section 3.8)
        if constexpr (std::is_same<ZS, SS>::value && (ZS::N == 16 || ZS::N == 32 || ZS::N == 64)) {
            constexpr int P = plane_group<ZS>();
            constexpr int MBP = (sizeof(T) == 8 && ZS::N == 32) ? 3 : 1024 / (ZS::T * ZS::N * P);
            e.launch[PK_PLANE] = launch_plane<ZS, T, P, MBP>;
            // the 2-D convolution of whole images: the plane kernel's CTA shape and register budget
            e.launch[PK_PLANE_CONV] = launch_plane_conv<ZS, T, P, MBP>;
        }
    }
    // fused two-pass kernels: the contiguous role is re-tiled so that both roles fill the same CTA
    constexpr int NT = SS::T * Y::C, NTP = SS::T * PEER::C;
    static_assert(NT % ZS::T == 0 && NTP % ZS::T == 0, "strided CTA size must be a multiple of the contiguous line's thread count");
    e.f_zC = NT / ZS::T;
    e.f_zCp = NTP / ZS::T;
    constexpr int H1 = (FH & 1) ? 1 : 0, H2 = (FH & 1) ? 2 : 0;
    constexpr bool ZL = (FH & 2) != 0 && ZS::T % 32 == 0 && NT / ZS::T <= 15;
    constexpr bool ZLp = (FH & 2) != 0 && ZS::T % 32 == 0 && NTP / ZS::T <= 15;
    // first-role flavour (intermediate written with evict_last) and second-role flavour (everything evict_first)
    using OZ = TileOp<ZS, T, NT / ZS::T, MAP_T, MAP_T, false, false, false, false, false, H1, H2, false, ZL>;
    using OZ2 = TileOp<ZS, T, NT / ZS::T, MAP_T, MAP_T, false, false, false, false, false, H1, H1, false, ZL>;
    using OZp = TileOp<ZS, T, NTP / ZS::T, MAP_T, MAP_T, false, false, false, false, false, H1, H2, false, ZLp>;
    using OY = TileOp<SS, T, Y::C, MAP_C, MAP_C, false, false, false, false, false, H1, H2>;
    using OY2 = TileOp<SS, T, Y::C, MAP_C, MAP_C, false, false, false, false, false, H1, H1>;
    using OYco = TileOp<SS, T, PEER::C, MAP_C, MAP_C, false, false, true, false, false, H1, 0>;
    using OYci = TileOp<SS, T, Y::C, MAP_C, MAP_C, false, true, false, false, false, H1, H2>;
    e.fused[FK_ZY] = fused_if_fits<OZ, OY2, T, Y::MB>();
    e.fused[FK_ZY_CO] = fused_if_fits<OZp, OYco, T, PEER::MB>();
    e.fused[FK_YZ] = fused_if_fits<OY, OZ2, T, Y::MB>();
    e.fused[FK_YZ_CI] = YCI::C == Y::C ? fused_if_fits<OYci, OZ2, T, Y::MB>() : nullptr;   // (the roles share Y's tile)
    // whole forward transform of a device in one kernel: needs the X role to fill the peer-store CTA shape
    e.fused3 = nullptr; e.fused_yx = nullptr;
    if constexpr (XS::T * X::C == NTP) {
        using OX = TileOp<XS, T, X::C, MAP_C, MAP_T, false, false, false, false>;
        if constexpr (roles_smem<OZp, OYco, OX>() <= SMEM_OPTIN_MAX) e.fused3 = launch_fused3<OZp, OYco, OX, T, (PEER::MB < X::MB ? PEER::MB : X::MB)>;
        if constexpr (roles_smem<OYco, OX>() <= SMEM_OPTIN_MAX) e.fused_yx = launch_fused_yx<OYco, OX, T, (PEER::MB < X::MB ? PEER::MB : X::MB)>;
    }
    return e;
}

}  // namespace dfft
