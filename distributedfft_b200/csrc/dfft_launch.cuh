// dfft_launch.cuh -- launch set-up shared by every pass-kernel launcher (dfft_kernels_inst.cuh, dfft_kernels_generic.cu,
// dfft_kernels_tma.cu).  The kernels are persistent: a grid of at most one wave of resident CTAs loops over the work units.
#pragma once
#include <atomic>
#include <cuda_runtime.h>

namespace dfft {

// Raises Kern's dynamic shared-memory limit to `bytes` on the calling thread's current device, once per (Kern, device).  The
// limit belongs to the device's copy of the function: a process driving several devices needs one call on each
template <auto Kern> cudaError_t smem_optin(size_t bytes)
{
    static std::atomic<bool> done[64];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess || done[dev & 63].load()) return e;
    e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) done[dev & 63].store(true);
    return e;
}

// CTAs of a persistent grid: min(sm_count * min(occ, cap), work); cap <= 0 leaves occ as it is.  0 when there is no work
inline long long grid_for(int sm_count, int occ, int cap, long long work)
{
    if (work <= 0) return 0;
    if (cap > 0 && occ > cap) occ = cap;
    const long long grid = (long long)sm_count * occ;
    return grid < work ? grid : work;
}

// grid of Kern launched with `threads` threads and `smem` bytes of dynamic shared memory over `work` units: the opt-in and the
// resident CTAs per SM, both once per (Kern, device), then grid_for.  For kernels whose block size and shared memory are fixed
// at compile time; grid = 0: nothing to launch
template <auto Kern> cudaError_t resident_grid(int threads, size_t smem, int cap, long long work, int sm_count, long long& grid)
{
    static std::atomic<int> occ_cache[64];
    grid = 0;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    int occ = occ_cache[dev & 63].load();
    if (occ == 0) {
        if ((e = smem_optin<Kern>(smem)) != cudaSuccess) return e;
        if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, Kern, threads, smem)) != cudaSuccess) return e;
        if (occ < 1) return cudaErrorLaunchOutOfResources;
        occ_cache[dev & 63].store(occ);
    }
    grid = grid_for(sm_count, occ, cap, work);
    return cudaSuccess;
}

}  // namespace dfft
