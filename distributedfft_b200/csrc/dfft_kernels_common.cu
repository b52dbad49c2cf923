// size table lookup, twiddle tables, and the element-wise helper kernels of the staged mode
#include <cmath>
#include <cstdlib>
#include <mutex>
#include "dfft_kernels.cuh"

namespace dfft {

void register_f64(std::vector<SizeEntry>& v);
void register_f32(std::vector<SizeEntry>& v);

static std::vector<SizeEntry>& table()
{
    static std::vector<SizeEntry> t;
    static std::once_flag once;
    std::call_once(once, [] { register_f64(t); register_f32(t); });
    return t;
}

const SizeEntry* find_size_entry(int N, int prec)
{
    const char* gen = getenv("DFFT_GENERIC");
    if (gen && atoi(gen) != 0) return generic_size_entry(N, prec);
    const char* env = getenv("DFFT_VARIANT");
    const int want = env ? atoi(env) : 0;
    const SizeEntry* def = nullptr;
    for (const SizeEntry& e : table()) {
        if (e.N != N || e.prec != prec) continue;
        if (e.variant == want) return &e;
        if (e.variant == 0) def = &e;
    }
    if (!def) return generic_size_entry(N, prec);
    return def;
}

// fft_plane_kernel against the separate X and Y passes, per (N, precision), from csrc/tools/lines3d_bench.py on H100
// (DESIGN.md section 7): true = the plane kernel is the default of the 3-D lines plans for that shape
static const struct { int N, prec; bool use; } kPlaneUse[] = {
    {16, 0, true}, {32, 0, true}, {64, 0, true}, {16, 1, true}, {32, 1, true}, {64, 1, true},
};

bool plane_default(int N, int prec)
{
    for (const auto& u : kPlaneUse)
        if (u.N == N && u.prec == prec) return u.use;
    return false;
}

// fft_plane_conv_kernel against the three passes X, XCONV, inverse X, per (N, precision), from
// csrc/tools/lines_conv_bench.py --dims 2 on H100 (DESIGN.md section 7): true = the default of the 2-D convolve lines plans
static const struct { int N, prec; bool use; } kPlaneConvUse[] = {
    {16, 0, true}, {32, 0, true}, {64, 0, true}, {16, 1, true}, {32, 1, true}, {64, 1, true},
};

bool plane_conv_default(int N, int prec)
{
    for (const auto& u : kPlaneConvUse)
        if (u.N == N && u.prec == prec) return u.use;
    return false;
}

void list_sizes(int prec, std::vector<int>& out)
{
    out.clear();
    for (const SizeEntry& e : table())
        if (e.prec == prec && e.variant == 0) out.push_back(e.N);
}

template <typename T> std::vector<cx<T>> build_lut(int nstages, const int* rad)
{
    std::vector<cx<T>> lut;
    long long ns = rad[0];
    const long double two_pi = 6.283185307179586476925286766559005768L;
    for (int s = 1; s < nstages; s++) {
        const int R = rad[s];
        for (int m = 1; m < R; m++)
            for (long long k = 0; k < ns; k++) {
                long double a = -two_pi * (long double)((k * m) % (ns * R)) / (long double)(ns * R);
                cx<T> w;
                w.x = (T)cosl(a);
                w.y = (T)sinl(a);
                lut.push_back(w);
            }
        ns *= R;
    }
    // padded so that the kernels' 16-byte-granular TMA bulk copy never reads past the allocation
    cx<T> zero; zero.x = 0; zero.y = 0;
    lut.push_back(zero); lut.push_back(zero);
    return lut;
}
template std::vector<cx<double>> build_lut<double>(int, const int*);
template std::vector<cx<float>> build_lut<float>(int, const int*);

// Row-granular per-destination pack / unpack: the restated index map of
// 3dmpifft_opt/include/kernel_func.cpp:73-100 (natural [x][y][z] <-> [q][x][y mod yd][z]).
// Used only by the staged (stage-by-stage, reference-like) mode; the production path folds this
// map into the Y-pass store / load.  One 16-byte vector per thread step, rows stay contiguous.
template <typename V>
__global__ void pack_rows_kernel(const V* __restrict__ in, V* __restrict__ out, long long x_size, long long n1,
                                 long long row_vecs, int P, int forward)
{
    const long long yd = (n1 + P - 1) / P, y_last = n1 - (P - 1) * yd;
    const long long rows = x_size * n1;
    for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
        const long long x = row / n1, y = row - x * n1;
        const long long q = y / yd;
        const long long w = (q == P - 1) ? y_last : yd;
        const long long nat = row * row_vecs;
        const long long pk = (x_size * yd * q + x * w + (y - q * yd)) * row_vecs;
        const V* src = forward ? in + nat : in + pk;
        V* dst = forward ? out + pk : out + nat;
        for (long long i = threadIdx.x; i < row_vecs; i += blockDim.x) dst[i] = src[i];
    }
}

cudaError_t launch_pack_rows(const void* in, void* out, int elem_bytes, long long x_size, long long n1, long long n2,
                             int P, int forward, int sm_count, cudaStream_t st)
{
    const long long rows = x_size * n1;
    if (rows == 0) return cudaSuccess;
    long long grid = (long long)sm_count * 8;
    if (grid > rows) grid = rows;
    if (elem_bytes == 16) {
        pack_rows_kernel<double2><<<(unsigned)grid, 256, 0, st>>>((const double2*)in, (double2*)out, x_size, n1, n2, P, forward);
    } else {
        pack_rows_kernel<float2><<<(unsigned)grid, 256, 0, st>>>((const float2*)in, (float2*)out, x_size, n1, n2, P, forward);
    }
    return cudaGetLastError();
}

}  // namespace dfft
