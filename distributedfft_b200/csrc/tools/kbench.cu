// kbench.cu -- developer micro-benchmark for the pass kernels (not part of the product path).
// Runs each pass variant on a 512^3-sized buffer, checks it on a plane-wave input (FFT of
// e^{2 pi i f n/N} is N at bin f) and prints time / achieved GB/s.
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>
#include <string>
#include "../fft_passes.cuh"

using namespace dfft;

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

template <class S> std::vector<double2> make_lut()
{
    std::vector<double2> lut(S::lut_size() > 0 ? S::lut_size() : 1);
    for (int s = 1; s < S::NSTAGES; s++) {
        int RAD = S::rad(s), NS = S::ns(s), off = S::lut_off(s);
        for (int m = 1; m < RAD; m++)
            for (int k = 0; k < NS; k++) {
                long double a = -2.0L * 3.14159265358979323846264338327950288L * (long double)(k * m) / (long double)(NS * RAD);
                lut[off + (m - 1) * NS + k] = make_double2((double)cosl(a), (double)sinl(a));
            }
    }
    return lut;
}

// fill: element (line index derived from strides) = plane wave with frequency f = (line % N)
__global__ void fill_wave(double2* buf, long long nlines, int N, long long line_stride_a, long long line_stride_b, int lines_b, long long es)
{
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    long long total = nlines * N;
    if (i >= total) return;
    long long line = i / N; int e = (int)(i % N);
    long long a = line / lines_b, b = line % lines_b;
    int f = (int)(line % N);
    double ang = 2.0 * M_PI * (double)((long long)f * e % N) / N;
    buf[a * line_stride_a + b * line_stride_b + (long long)e * es] = make_double2(cos(ang), sin(ang));
}
__global__ void check_wave(const double2* buf, long long nlines, int N, long long line_stride_a, long long line_stride_b, int lines_b, long long es, double* maxerr)
{
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    long long total = nlines * N;
    if (i >= total) return;
    long long line = i / N; int e = (int)(i % N);
    long long a = line / lines_b, b = line % lines_b;
    int f = (int)(line % N);
    double2 v = buf[a * line_stride_a + b * line_stride_b + (long long)e * es];
    double ex = (e == f) ? (double)N : 0.0;
    double err = fmax(fabs(v.x - ex), fabs(v.y));
    if (err > 1e-9) atomicMax((unsigned long long*)maxerr, (unsigned long long)__double_as_longlong(err));
}

struct Result { std::string name; float ms; double gbs; double err; int regs; size_t smem; int occ; };
static std::vector<Result> results;
static double2 *d_a, *d_b; static double* d_err;
static int NX = 512, NY = 512, NZ = 512;   // cube edge = transform length of the variant set being run
static int g_sms = 132;
static int g_only = -1, g_idx = 0;

template <class S, int C, int MAPIN, int MAPOUT, bool TWREG, bool PREFETCH, int MINB, bool PP = true>
void run_variant(const char* name, int pass /*0 Z,1 Y,2 X*/, int ctas_per_sm)
{
    using T = double;
    if (g_only >= 0 && g_idx++ != g_only) return;
    if (g_only < 0) g_idx++;
    auto kern = fft_tile_kernel<S, T, C, MAPIN, MAPOUT, TWREG, false, false, MINB, PP, PREFETCH>;
    using SM = TileSmem<S, T, C, PP>;
    size_t smem = SM::bytes(false) + TileOp<S, T, C, MAPIN, MAPOUT, TWREG, false, false, PP, PREFETCH>::stage_bytes;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaFuncAttributes fa; CK(cudaFuncGetAttributes(&fa, kern));
    int occ = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, S::T * C, smem));
    static double2* d_lut = nullptr; static int lut_for = 0;
    auto lut = make_lut<S>();
    if (d_lut) cudaFree(d_lut);
    CK(cudaMalloc(&d_lut, lut.size() * sizeof(double2)));
    CK(cudaMemcpy(d_lut, lut.data(), lut.size() * sizeof(double2), cudaMemcpyHostToDevice)); (void)lut_for;

    TileArgs<T> A{}; A.lut = d_lut; A.scale = 1.0;
    const long long plane = (long long)NY * NZ;
    long long nlines; long long lsa, lsb; int lb; long long es_in; long long osa, osb; int olb; long long es_out;
    if (pass == 0) { // Z: lines (x,y) contiguous z
        A.in = d_a; A.out = d_a;
        nlines = (long long)NX * NY; A.G = (int)((nlines + C - 1) / C); A.W = (int)nlines; A.ntiles = A.G;
        A.ia = Affine{0, (long long)C * NZ, NZ, 1}; A.oa = A.ia;
        lsa = 0; lsb = NZ; lb = (int)nlines; es_in = 1; osa = lsa; osb = lsb; olb = lb; es_out = 1;
    } else if (pass == 1) { // Y: tile (x, zgroup): rows y stride NZ
        A.in = d_a; A.out = d_a;
        A.G = (NZ + C - 1) / C; A.W = NZ; A.ntiles = (long long)NX * A.G;
        A.ia = Affine{plane, C, 1, NZ}; A.oa = A.ia;
        nlines = (long long)NX * NZ; lsa = plane; lsb = 1; lb = NZ; es_in = NZ; osa = lsa; osb = lsb; olb = lb; es_out = NZ;
    } else { // X: in [x][y][z] -> out [y][z][x]; tile (y, zgroup)
        A.in = d_a; A.out = d_b;
        A.G = (NZ + C - 1) / C; A.W = NZ; A.ntiles = (long long)NY * A.G;
        A.ia = Affine{NZ, C, 1, plane};
        A.oa = Affine{(long long)NZ * NX, (long long)C * NX, NX, 1};
        nlines = (long long)NY * NZ; lsa = NZ; lsb = 1; lb = NZ; es_in = plane; osa = (long long)NZ * NX; osb = NX; olb = NZ; es_out = 1;
    }
    int grid = g_sms * (ctas_per_sm > 0 ? ctas_per_sm : occ);
    if (grid > A.ntiles) grid = (int)A.ntiles;
    long long total = nlines * S::N;
    fill_wave<<<(unsigned)((total + 255) / 256), 256>>>(d_a, nlines, S::N, lsa, lsb, lb, es_in);
    CK(cudaMemset(d_err, 0, 8));
    kern<<<grid, S::T * C, smem>>>(A);
    CK(cudaGetLastError());
    check_wave<<<(unsigned)((total + 255) / 256), 256>>>(pass == 2 ? d_b : d_a, nlines, S::N, osa, osb, olb, es_out, d_err);
    CK(cudaDeviceSynchronize());
    double err; CK(cudaMemcpy(&err, d_err, 8, cudaMemcpyDeviceToHost));
    // timing: data (2 GiB) >> L2, so no flush needed
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int i = 0; i < 2; i++) kern<<<grid, S::T * C, smem>>>(A);
    const int iters = 5;
    cudaEventRecord(e0);
    for (int i = 0; i < iters; i++) kern<<<grid, S::T * C, smem>>>(A);
    cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= iters;
    double bytes = 2.0 * 16.0 * (double)total;
    results.push_back({name, ms, bytes / ms * 1e-6, err, fa.numRegs, smem, occ});
    printf("[%2d] %-44s pass=%d grid=%5d thr=%4d regs=%3d smem=%6zu occ=%d  %.3f ms  %.0f GB/s  err=%.2e\n", g_idx - 1, name, pass, grid, S::T * C, fa.numRegs, smem, occ, ms, bytes / ms * 1e-6, err);
    fflush(stdout);
}


// pure data-movement twin of the strided passes: same tile/thread map, no FFT
template <int C, int TT, int R>
__global__ void __launch_bounds__(C* TT) tile_copy_kernel(const TileArgs<double> A, int N)
{
    const int c = threadIdx.x % C, t = threadIdx.x / C;
    for (long long tile = blockIdx.x; tile < A.ntiles; tile += gridDim.x) {
        const long long a = tile / A.G; const int b = (int)(tile - a * A.G);
        const double2* p = A.in + a * A.ia.SA + b * A.ia.SB + c * A.ia.cs;
        double2* q = A.out + a * A.oa.SA + b * A.oa.SB + c * A.oa.cs;
        for (int e0 = 0; e0 < N; e0 += TT * R) {
            double2 v[R];
#pragma unroll
            for (int u = 0; u < R; u++) v[u] = __ldcg(p + (long long)(e0 + t + u * TT) * A.ia.es);
#pragma unroll
            for (int u = 0; u < R; u++) __stcg(q + (long long)(e0 + t + u * TT) * A.oa.es, v[u]);
        }
    }
}
template <int C, int TT, int R>
void run_copy(const char* name, int pattern /*1 Y-like, 2 X-like*/, bool inplace, int cps)
{
    if (g_only >= 0 && g_idx++ != g_only) return;
    if (g_only < 0) g_idx++;
    TileArgs<double> A{};
    const long long plane = (long long)NY * NZ;
    A.in = d_a; A.out = inplace ? d_a : d_b;
    A.G = NZ / C; A.W = NZ;
    if (pattern == 1) { A.ntiles = (long long)NX * A.G; A.ia = Affine{plane, C, 1, NZ}; }
    else { A.ntiles = (long long)NY * A.G; A.ia = Affine{NZ, C, 1, plane}; }
    A.oa = A.ia;
    int grid = g_sms * cps; if (grid > A.ntiles) grid = (int)A.ntiles;
    auto kern = tile_copy_kernel<C, TT, R>;
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int i = 0; i < 2; i++) kern<<<grid, C * TT>>>(A, 512);
    cudaEventRecord(e0);
    for (int i = 0; i < 5; i++) kern<<<grid, C * TT>>>(A, 512);
    cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
    float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 5;
    double bytes = 2.0 * 16.0 * (double)NX * NY * NZ;
    printf("[%2d] COPY %-30s pattern=%d inplace=%d grid=%5d thr=%4d  %.3f ms  %.0f GB/s\n", g_idx - 1, name, pattern, (int)inplace, grid, C * TT, ms, bytes / ms * 1e-6);
    fflush(stdout);
}

__global__ void copy_kernel(const double2* __restrict__ in, double2* __restrict__ out, long long n)
{
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    long long stride = (long long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) __stcg(out + i, __ldcg(in + i));
}

int main(int argc, char** argv)
{
    int N = argc > 1 ? atoi(argv[1]) : 512;
    if (argc > 2) g_only = atoi(argv[2]);
    NX = NY = NZ = N;
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    g_sms = prop.multiProcessorCount;
    printf("device %s sms=%d  cube %d^3 fp64\n", prop.name, g_sms, N);
    size_t n = (size_t)NX * NY * NZ;
    CK(cudaMalloc(&d_a, n * sizeof(double2))); CK(cudaMalloc(&d_b, n * sizeof(double2))); CK(cudaMalloc(&d_err, 8));
    if (g_only < 0) {   // copy roofline reference
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        copy_kernel<<<g_sms * 8, 512>>>(d_a, d_b, (long long)n);
        cudaEventRecord(e0);
        for (int i = 0; i < 5; i++) copy_kernel<<<g_sms * 8, 512>>>(d_a, d_b, (long long)n);
        cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
        float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 5;
        printf("copy: %.3f ms  %.0f GB/s\n", ms, 2.0 * 16.0 * n / ms * 1e-6);
    }
#define VP(S, C, MI, MO, TW, PF, MB, PP, pass, cps) run_variant<S, C, MI, MO, TW, PF, MB, PP>(#S " C" #C " tw" #TW " pf" #PF " mb" #MB " pp" #PP, pass, cps)
    if (N == 512) {
        using S512 = Sched<512, 8, 8, 8, 8>;
        using S512b = Sched<512, 16, 8, 8, 8>;
        VP(S512, 2, MAP_T, MAP_T, true, false, 4, true, 0, 0);
        VP(S512, 2, MAP_T, MAP_T, true, true, 3, true, 0, 0);
        VP(S512b, 8, MAP_C, MAP_C, false, false, 2, false, 1, 0);
        VP(S512b, 8, MAP_C, MAP_T, false, false, 2, false, 2, 0);
    } else if (N == 1024) {
        using S1024 = Sched<1024, 16, 16, 8, 8>;
        using S1024x = Sched<1024, 8, 8, 8, 8, 2>;
        // Z
        VP(S1024, 2, MAP_T, MAP_T, false, false, 4, true, 0, 0);    // current
        VP(S1024, 2, MAP_T, MAP_T, false, false, 4, false, 0, 0);
        VP(S1024, 1, MAP_T, MAP_T, false, false, 8, true, 0, 0);
        VP(S1024, 4, MAP_T, MAP_T, false, false, 2, false, 0, 0);
        VP(S1024x, 1, MAP_T, MAP_T, true, false, 4, true, 0, 0);
        VP(S1024x, 1, MAP_T, MAP_T, false, false, 4, true, 0, 0);
        VP(S1024x, 2, MAP_T, MAP_T, false, false, 2, true, 0, 0);
        VP(S1024, 2, MAP_T, MAP_T, false, true, 3, false, 0, 0);
        // Y
        VP(S1024, 4, MAP_C, MAP_C, false, false, 2, false, 1, 0);   // v0
        VP(S1024, 8, MAP_C, MAP_C, false, false, 1, false, 1, 0);   // v1
        VP(S1024x, 4, MAP_C, MAP_C, false, false, 2, false, 1, 0);
        VP(S1024x, 8, MAP_C, MAP_C, false, false, 1, false, 1, 0);
        VP(S1024, 4, MAP_C, MAP_C, false, false, 3, false, 1, 0);
        // X
        VP(S1024, 4, MAP_C, MAP_T, false, false, 2, false, 2, 0);
        VP(S1024, 8, MAP_C, MAP_T, false, false, 1, false, 2, 0);
        VP(S1024x, 4, MAP_C, MAP_T, false, false, 2, false, 2, 0);
        VP(S1024x, 8, MAP_C, MAP_T, false, false, 1, false, 2, 0);
    } else if (N == 768) {
        using S768 = Sched<768, 12, 4, 4, 4, 4, 3>;
        using S768b = Sched<768, 24, 8, 8, 4, 3>;
        using S768c = Sched<768, 6, 3, 2, 2, 2, 2, 2, 2, 2, 2>;
        (void)sizeof(S768c);
        // Z
        VP(S768, 2, MAP_T, MAP_T, false, false, 4, true, 0, 0);     // current
        VP(S768, 2, MAP_T, MAP_T, false, false, 4, false, 0, 0);
        VP(S768, 4, MAP_T, MAP_T, false, false, 2, false, 0, 0);
        VP(S768, 1, MAP_T, MAP_T, false, false, 8, true, 0, 0);
        VP(S768b, 4, MAP_T, MAP_T, false, false, 2, false, 0, 0);
        VP(S768b, 2, MAP_T, MAP_T, false, false, 4, true, 0, 0);
        VP(S768b, 8, MAP_T, MAP_T, false, false, 1, false, 0, 0);
        // Y
        VP(S768, 4, MAP_C, MAP_C, false, false, 2, false, 1, 0);    // current
        VP(S768, 8, MAP_C, MAP_C, false, false, 1, false, 1, 0);
        VP(S768b, 4, MAP_C, MAP_C, false, false, 2, false, 1, 0);
        VP(S768b, 8, MAP_C, MAP_C, false, false, 1, false, 1, 0);
        VP(S768b, 8, MAP_C, MAP_C, false, false, 2, false, 1, 0);
        // X
        VP(S768, 4, MAP_C, MAP_T, false, false, 2, false, 2, 0);
        VP(S768, 8, MAP_C, MAP_T, false, false, 1, false, 2, 0);
        VP(S768b, 4, MAP_C, MAP_T, false, false, 2, false, 2, 0);
        VP(S768b, 8, MAP_C, MAP_T, false, false, 1, false, 2, 0);
        VP(S768b, 8, MAP_C, MAP_T, false, false, 2, false, 2, 0);
    }
    return 0;
}
