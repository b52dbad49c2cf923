// dfft_kernels.cuh -- table of pre-instantiated pass kernels, one entry per (length, precision).
// The reference compiles one kernel per axis at plan time with hiprtc
// (templateFFT/src/templateFFT.cpp:5614-5752); here the supported lengths are instantiated ahead
// of time for sm_90a and looked up at plan time.
#pragma once
#include <cuda_runtime.h>
#include <vector>
#include "fft_passes.cuh"
#include "fft_real.cuh"
#include "fft_plane.cuh"

namespace dfft {

enum PassKind {
    PK_Z = 0,      // contiguous lines, MAP_T -> MAP_T
    PK_Y,          // strided, MAP_C -> MAP_C
    PK_Y_CO,       // + chunked (pack / peer) store
    PK_Y_CI,       // + chunked (unpack) load
    PK_XF,         // strided load, transposed contiguous store (MAP_C -> MAP_T)
    PK_XB,         // contiguous load, strided store (MAP_T -> MAP_C)
    PK_XB_CO,      // + chunked (peer) store
    PK_XF_TW,      // PK_XF + four-step twiddle epilogue (first pass of a long 1-D transform)
    PK_Z_R2C,      // real lines -> half spectra, two lines per complex transform (fft_real.cuh; args = RealZArgs)
    PK_Z_C2R,      // half spectra -> real lines (fft_real.cuh; args = RealZArgs)
    PK_XCONV,      // spectral convolution along x: forward, multiply, inverse in one column pass (fft_conv_kernel; args = ConvArgs),
                   // strided local configuration, local store
    PK_XCONV_CO,   // + chunked (peer) store split by xd, in the peer-store configuration
    // the lines engine's whole-plane and whole-line kernels, on the contiguous schedule; default entries only, else nullptr
    PK_PLANE,          // X + Y passes of whole N x N planes in one kernel (fft_plane_kernel; args = PlaneArgs); N = 16, 32, 64 only
                       // (both roles share one schedule there)
    PK_PLANE_CONV,     // 2-D convolution of whole N x N images in one kernel (fft_plane_conv_kernel; args = PlaneConvArgs); set where
                       // PK_PLANE is
    PK_LINE_CONV,      // 1-D convolution of contiguous lines in one pass (fft_line_conv_kernel; args = LineConvArgs)
    PK_LINE_CONV_R2C,  // + real lines, two per complex transform (fft_line_conv_r2c_kernel; args = RealLineConvArgs)
    PK_COUNT
};

typedef cudaError_t (*PassLaunchFn)(const void* tile_args, int sm_count, cudaStream_t stream);

// two dependent passes over the same planes in one persistent kernel (fft_fused2_kernel)
enum FusedKind {
    FK_ZY = 0,     // forward t0: Z then Y, natural store
    FK_ZY_CO,      // forward t0 + t1 (+ t2 over NVLink): Z then Y with the chunked (pack / peer) store
    FK_YZ,         // backward t0: Y then Z
    FK_YZ_CI,      // backward t1 + t0: Y with the chunked (unpack) load, then Z
    FK_COUNT
};
typedef cudaError_t (*FusedLaunchFn)(const void* args_a, const void* args_b, const FusedCtl* ctl, int sm_count, cudaStream_t stream);
// forward t0..t3 of one device in one kernel (fft_fused3_kernel): Z, Y with peer stores, X behind per-part arrival flags
// send side (Y pass of part k, peer stores) and receive side (X pass of part k-1) of the exchange in one kernel (fft_fused_yx_kernel)
typedef cudaError_t (*FusedYxLaunchFn)(const void* args_y, const void* args_x, const YxCtl* ctl, int sm_count, cudaStream_t stream);
typedef cudaError_t (*Fused3LaunchFn)(const void* args_z, const void* args_y, const void* args_x, const Fused3Ctl* ctl, int sm_count, cudaStream_t stream);

struct SizeEntry {
    int N;
    int variant;          // 0 = default; > 0 = alternate tuning of the same length, selected with DFFT_VARIANT (experiments)
    int prec;             // 0 = double, 1 = float
    int z_C, s_C, p_C, x_C;   // lines per tile: contiguous (Z), strided local (Y), strided with peer/packed store, X passes
    int ci_C, xo_C;           // lines per tile of the Y pass with the chunked (unpack) load and of the X pass with the chunked store:
                              // s_C and x_C, halved where that tile, its twiddles and the chunk tables would not fit in one block's
                              // shared memory (4096-point fp64); p_C is chosen the same way
    int z_nstages, z_rad[24];
    int s_nstages, s_rad[24];
    int x_nstages, x_rad[24];
    PassLaunchFn launch[PK_COUNT];
    int f_zC, f_zCp;      // lines per contiguous tile inside the fused kernels (same CTA size as the strided role; p: peer-store kind)
    FusedLaunchFn fused[FK_COUNT];   // valid for square planes (N1 == N2 == N): both roles come from this entry
    FusedYxLaunchFn fused_yx;        // Y (peer-store configuration) + X roles of this entry in one kernel; nullptr unless both fill the same CTA
    Fused3LaunchFn fused3;           // same restriction, and the X configuration must fill the same CTA as the peer-store Y role (else nullptr)
    const void* gen;      // run-time schedule (GenSched) of a generic-length entry, nullptr for tuned lengths
};

// whether fft_plane_kernel is the default for (N, prec) (measured against the two separate passes, dfft_kernels_common.cu)
bool plane_default(int N, int prec);
// whether fft_plane_conv_kernel is the default of the 2-D convolve lines plans for (N, prec) (measured against the three passes)
bool plane_conv_default(int N, int prec);

// TMA-pipelined pass kernels (fft_tma.cuh), instantiated for the lengths whose C-line tile fills a 64 KB ring slot
typedef cudaError_t (*TmaLaunchFn)(int mode, const void* tma_args, const void* map_in, const void* map_out, int sm_count, cudaStream_t stream);
// forward t0 of square planes in one kernel (fft_tma_fused_zy_kernel): args = TmaFusedArgs<T>, map_mid = 3-D map of the intermediate
typedef cudaError_t (*TmaFusedLaunchFn)(const void* fused_args, const FusedCtl* ctl, const void* map_mid, int sm_count, cudaStream_t stream);
constexpr int TMA_USE_ZY = 4;   // TmaEntry::use bit of the fused forward t0
struct TmaEntry {
    int N, prec;
    int C;                 // lines / columns per tile
    int rows;              // rows per tensor copy (transform length split into N / rows boxes)
    int nstages, rad[24];  // radix schedule (its twiddle table: build_lut)
    TmaLaunchFn launch;
    TmaFusedLaunchFn fused_zy;   // nullptr: no fused forward t0 for this length
    unsigned use;          // bit m set: mode m (TMA_Z, TMA_Y, TMA_XF, TMA_XB) beats the register-staged kernel
                           // (per-pass sweeps, dfft_kernels_tma.cu); DFFT_TMA=2 uses every mode, DFFT_TMA=0 none;
                           // bit TMA_USE_ZY: fused_zy is the default forward t0 of one-device plans
};
const TmaEntry* find_tma_entry(int N, int prec);   // nullptr: no instantiation, driver too old, or DFFT_TMA=0
int tma_encode_3d(void* map, void* base, int prec, long long d0, long long d1, long long d2, long long s1, long long s2, int b0, int b1, int b2);

// tuned entry if the length is in the table, else a generic (run-time scheduled) entry for 2..13-smooth lengths,
// else nullptr.  DFFT_GENERIC=1 forces the generic kernel (tests).
const SizeEntry* find_size_entry(int N, int prec);
const SizeEntry* generic_size_entry(int N, int prec);
void list_sizes(int prec, std::vector<int>& out);

// twiddle table of a radix list, layout of Sched::lut_off(): per stage s >= 1,
// entry (m-1)*NS + k = e^{-2 pi i k m / (NS * RAD)}; evaluated in long double, rounded once.
template <typename T> std::vector<cx<T>> build_lut(int nstages, const int* rad);

// element-wise helpers (staged reference-like mode, tests)
cudaError_t launch_pack_rows(const void* in, void* out, int elem_bytes, long long x_size, long long n1, long long n2,
                             int P, int forward, int sm_count, cudaStream_t st);

}  // namespace dfft
