// Host side of the run-time-scheduled kernel (fft_generic.cuh): schedule construction for any
// 2..13-smooth length and a cache of SizeEntry records so the plan code treats them like tuned lengths.
#include <map>
#include <mutex>
#include "dfft_kernels.cuh"
#include "fft_generic.cuh"

namespace dfft {

// Radix schedule in the reference's manner (templateFFT/src/templateFFT.cpp:3956-3963 factor over 2..13,
// :4540-4550 merge three 2s into an 8 then two 2s into a 4, :4580-4588 descending radix order).
static bool make_generic_sched(int N, int prec, GenSched& g)
{
    if (N < 2) return false;
    int mult[14] = {0};
    int t = N;
    for (int p : {2, 3, 5, 7, 11, 13})
        while (t % p == 0) { t /= p; mult[p]++; }
    if (t != 1) return false;
    mult[8] = mult[2] / 3; mult[2] -= 3 * mult[8];
    mult[4] = mult[2] / 2; mult[2] -= 2 * mult[4];
    g = GenSched{};
    g.N = N;
    int ns = 1, off = 0;
    for (int r = 13; r >= 2; r--)
        for (int k = 0; k < mult[r]; k++) {
            if (g.nstages >= GEN_MAX_STAGES) return false;
            const int s = g.nstages++;
            g.rad[s] = r;
            g.ns[s] = ns;
            g.lut_off[s] = off;
            if (s > 0) off += (r - 1) * ns;
            ns *= r;
        }
    const size_t esz = prec == 0 ? 16 : 8;
    const size_t budget = 192 * 1024;
    const size_t line2 = 2 * (size_t)N * esz;   // two ping-pong copies of one line
    if (line2 > 200 * 1024) return false;
    size_t C = budget / line2;
    g.C = (int)(C < 1 ? 1 : (C > 8 ? 8 : C));
    return true;
}

template <typename T, int MI, int MO, bool CI, bool CO>
static cudaError_t launch_generic(const void* vargs, int sm_count, cudaStream_t st)
{
    const TileArgs<T>& a = *reinterpret_cast<const TileArgs<T>*>(vargs);
    if (!a.gen) return cudaErrorInvalidValue;
    const GenSched& g = *reinterpret_cast<const GenSched*>(a.gen);
    auto kern = fft_generic_kernel<T, MI, MO, CI, CO>;
    const size_t smem = 2 * (size_t)g.C * g.N * sizeof(cx<T>);
    static std::mutex mu;
    static size_t attr_set[64] = {0};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    {
        std::lock_guard<std::mutex> lk(mu);
        if (attr_set[dev & 63] < smem) {
            e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024));
            if (e != cudaSuccess) return e;
            attr_set[dev & 63] = 200 * 1024;
        }
    }
    if (a.ntiles <= 0) return cudaSuccess;
    int occ = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, GEN_THREADS, smem);
    if (e != cudaSuccess) return e;
    if (occ < 1) return cudaErrorLaunchOutOfResources;
    if (a.max_ctas_per_sm > 0 && occ > a.max_ctas_per_sm) occ = a.max_ctas_per_sm;
    long long grid = (long long)sm_count * occ;
    if (grid > a.ntiles) grid = a.ntiles;
    kern<<<(unsigned)grid, GEN_THREADS, smem, st>>>(a, g);
    return cudaGetLastError();
}

// real-data passes (fft_generic_r2c_kernel / fft_generic_c2r_kernel): vargs is a RealZArgs<T>, a tile is G.C line pairs
template <typename T, bool INV>
static cudaError_t launch_generic_real(const void* vargs, int sm_count, cudaStream_t st)
{
    const RealZArgs<T>& a = *reinterpret_cast<const RealZArgs<T>*>(vargs);
    if (!a.t.gen) return cudaErrorInvalidValue;
    const GenSched& g = *reinterpret_cast<const GenSched*>(a.t.gen);
    auto kern = INV ? fft_generic_c2r_kernel<T> : fft_generic_r2c_kernel<T>;
    const size_t smem = 2 * (size_t)g.C * g.N * sizeof(cx<T>);
    static std::mutex mu;
    static size_t attr_set[64] = {0};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    {
        std::lock_guard<std::mutex> lk(mu);
        if (attr_set[dev & 63] < smem) {
            e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024));
            if (e != cudaSuccess) return e;
            attr_set[dev & 63] = 200 * 1024;
        }
    }
    if (a.t.ntiles <= 0) return cudaSuccess;
    int occ = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, GEN_THREADS, smem);
    if (e != cudaSuccess) return e;
    if (occ < 1) return cudaErrorLaunchOutOfResources;
    long long grid = (long long)sm_count * occ;
    if (grid > a.t.ntiles) grid = a.t.ntiles;
    kern<<<(unsigned)grid, GEN_THREADS, smem, st>>>(a, g);
    return cudaGetLastError();
}

template <typename T> static void fill_launchers(SizeEntry& e)
{
    e.launch[PK_Z] = launch_generic<T, MAP_T, MAP_T, false, false>;
    e.launch[PK_Y] = launch_generic<T, MAP_C, MAP_C, false, false>;
    e.launch[PK_Y_CO] = launch_generic<T, MAP_C, MAP_C, false, true>;
    e.launch[PK_Y_CI] = launch_generic<T, MAP_C, MAP_C, true, false>;
    e.launch[PK_XF] = launch_generic<T, MAP_C, MAP_T, false, false>;
    e.launch[PK_XB] = launch_generic<T, MAP_T, MAP_C, false, false>;
    e.launch[PK_XB_CO] = launch_generic<T, MAP_T, MAP_C, false, true>;
    e.launch[PK_XF_TW] = launch_generic<T, MAP_C, MAP_T, false, false>;   // the twiddle epilogue is a run-time switch (TileArgs::tw_n)
    // real lines of the lines engine; the 3-D R2C plan still refuses generic z lengths (plan_create)
    e.launch[PK_Z_R2C] = launch_generic_real<T, false>;
    e.launch[PK_Z_C2R] = launch_generic_real<T, true>;
}

const SizeEntry* generic_size_entry(int N, int prec)
{
    static std::mutex mu;
    static std::map<std::pair<int, int>, SizeEntry*> cache;
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find({N, prec});
    if (it != cache.end()) return it->second;
    GenSched* g = new GenSched;
    if (!make_generic_sched(N, prec, *g)) {
        delete g;
        cache[{N, prec}] = nullptr;
        return nullptr;
    }
    SizeEntry* e = new SizeEntry{};
    e->N = N; e->prec = prec; e->variant = 0;
    e->z_C = e->s_C = e->p_C = e->x_C = e->ci_C = e->xo_C = g->C;
    e->f_zC = e->f_zCp = 0;
    e->z_nstages = e->s_nstages = e->x_nstages = g->nstages;
    for (int s = 0; s < g->nstages; s++) e->z_rad[s] = e->s_rad[s] = e->x_rad[s] = g->rad[s];
    e->gen = g;
    if (prec == 0) fill_launchers<double>(*e);
    else fill_launchers<float>(*e);
    cache[{N, prec}] = e;
    return e;
}

}  // namespace dfft
