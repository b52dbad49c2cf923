/*
 * fft_mpi_3d_api.h -- header-only C++ shim that gives libdfft.so the reference's original names and
 * signatures (3dmpifft_opt/include/fft_mpi_3d_api.h:68-74, fft_mpi_common.h:15-22), so the reference
 * driver's call sequence (3dmpifft_opt/fftSpeed3d_c2c.cpp:42-102) compiles against it with
 * hip* -> cuda* as the only edit.  Error behaviour is the reference's: print and exit(EXIT_FAILURE).
 *
 * MPI_Comm: the reference takes an MPI communicator only to learn rank/size and to bootstrap; in a
 * single process (GPUs-per-rank mode, the only mode the reference's speedTest.sh exercises per node)
 * there is nothing to bootstrap, so when <mpi.h> is not included the shim defines MPI_Comm as an
 * int and ignores it.  Process-per-GPU programs use dfft_comm_create_bootstrap() directly.
 */
#ifndef DFFT_FFT_MPI_3D_API_SHIM_H
#define DFFT_FFT_MPI_3D_API_SHIM_H

#include <cstdio>
#include <cstdlib>
#include <mutex>

#include "dfft.h"

#define ALLOC_CPU DFFT_ALLOC_CPU
#define ALLOC_DEV DFFT_ALLOC_DEV
#define FORWARD DFFT_FORWARD
#define BACKWARD DFFT_BACKWARD

typedef double Complex[2];
typedef long long longInt64;

#ifndef MPI_VERSION
typedef int MPI_Comm;
#ifndef MPI_COMM_WORLD
#define MPI_COMM_WORLD 0
#endif
#endif

#define DFFT_CHECK(stmt)                                                                              \
    do {                                                                                              \
        int dfft_errno_ = (stmt);                                                                     \
        if (dfft_errno_ != 0) {                                                                       \
            fprintf(stderr, "[%s:%d] dfft call '%s' failed with %d: %s\n", __FILE__, __LINE__, #stmt, \
                    dfft_errno_, dfft_last_error());                                                  \
            exit(EXIT_FAILURE);                                                                       \
        }                                                                                             \
    } while (0)

/* the public part of the reference's plan struct (fft_mpi_3d_api.h:11-66) that callers touch */
typedef struct fft_mpi_3d_plan {
    int N[3];
    int locGPUIdx, devCountInNode, totalDevCount, globalDevIdx;
    bool isLastDevice, isInplace;
    longInt64 maxDataCountInDevice;
    Complex *inDev, *outDev, *bufferDev1, *bufferDev2, **nodeDataDev;
    int direction;
    dfft_plan impl;
    double t[5];
} * fft_mpi_3d_plan_p;

namespace dfft_shim {
inline dfft_comm& local_comm(int nranks)
{
    static std::mutex mu;
    static dfft_comm comm = nullptr;
    static int size = 0;
    std::lock_guard<std::mutex> lk(mu);
    if (nranks > 1 && (!comm || size != nranks)) {
        DFFT_CHECK(dfft_comm_create_local(nranks, &comm));
        size = nranks;
    }
    return comm;
}
inline int& device_count()   // device count chosen by the last fft_mpi_init (what an MPI_Comm would tell the reference)
{
    static int n = 1;
    return n;
}
}  // namespace dfft_shim

inline longInt64 getMaxDataCount(int n0, int n1, int n2, int totalDevCount, bool isLastDevice)
{
    return dfft_max_data_count(n0, n1, n2, totalDevCount, isLastDevice ? 1 : 0);
}

inline void fft_mpi_init(const longInt64* N, int iniDeviceNumInNode, MPI_Comm, int& newDeviceCount,
                         int& newDeviceCountInNode, longInt64 dataCountInNode[])
{
    DFFT_CHECK(dfft_init(N, iniDeviceNumInNode, &newDeviceCount, &newDeviceCountInNode, dataCountInNode));
    printf("allocate %d devices to node %d\n", newDeviceCountInNode, 0);                 /* api.cpp:270 */
    for (int i = 0; i < newDeviceCountInNode; ++i)
        printf("data count in device %d of node %d: %lld\n", i, 0, dataCountInNode[i]);  /* api.cpp:285 */
    if (newDeviceCount > 1) dfft_shim::local_comm(newDeviceCount);
    dfft_shim::device_count() = newDeviceCount;
}

inline void fft_mpi_cleanup(void) { dfft_cleanup(); }

inline longInt64 fft_mpi_local_size_3d(longInt64 n0, longInt64 n1, longInt64 n2, int totalDevCount, int devIdx,
                                       longInt64* local_n0, longInt64* local_0_start)
{
    return dfft_local_size_3d(n0, n1, n2, totalDevCount, devIdx, local_n0, local_0_start, nullptr, nullptr);
}

/* the reference's own declaration (fft_mpi_3d_api.h:73; never defined there): the slab of the calling rank, i.e. of device
 * 0 of the device count chosen by the last fft_mpi_init in this single-process build */
inline longInt64 fft_mpi_local_size_3d(longInt64 n0, longInt64 n1, longInt64 n2, MPI_Comm, longInt64* local_n0, longInt64* local_0_start)
{
    return dfft_local_size_3d(n0, n1, n2, dfft_shim::device_count(), 0, local_n0, local_0_start, nullptr, nullptr);
}

inline Complex* fft_mpi_alloc_local_memory(longInt64 count, int flag)
{
    void* p = dfft_alloc_local(count, flag, DFFT_DOUBLE);
    if (!p) {
        printf("Fail to allocate memory!\n");   /* api.cpp:226 */
        exit(EXIT_FAILURE);
    }
    return (Complex*)p;
}

inline fft_mpi_3d_plan_p fft_mpi_plan_dft_c2c_3d(longInt64 n0, longInt64 n1, longInt64 n2, Complex* in, Complex* out,
                                                 Complex** node_data, MPI_Comm, int devIdx, int devCountInNode,
                                                 int totalDevCount, int direction)
{
    fft_mpi_3d_plan_p plan = new fft_mpi_3d_plan();
    plan->N[0] = (int)n0; plan->N[1] = (int)n1; plan->N[2] = (int)n2;
    plan->direction = direction;
    plan->locGPUIdx = devIdx; plan->devCountInNode = devCountInNode; plan->totalDevCount = totalDevCount;
    plan->globalDevIdx = devIdx;
    plan->isLastDevice = devIdx == totalDevCount - 1;
    plan->maxDataCountInDevice = dfft_max_data_count(n0, n1, n2, totalDevCount, plan->isLastDevice);
    plan->inDev = in; plan->outDev = out;
    plan->isInplace = (out == nullptr || out == in);
    dfft_comm comm = totalDevCount > 1 ? dfft_shim::local_comm(totalDevCount) : nullptr;
    DFFT_CHECK(dfft_plan_c2c_3d(n0, n1, n2, in, out, comm, devIdx, totalDevCount, direction, DFFT_DOUBLE, DFFT_EXCHANGE_AUTO, &plan->impl));
    void *b1 = nullptr, *b2 = nullptr;
    DFFT_CHECK(dfft_plan_buffers(plan->impl, &b1, &b2));
    plan->bufferDev1 = (Complex*)b1; plan->bufferDev2 = (Complex*)b2;
    plan->nodeDataDev = node_data;
    if (node_data) node_data[devIdx] = plan->bufferDev1;   /* api.cpp:79-80 */
    return plan;
}

/* Real-to-complex (direction FORWARD: `in` = real x-slab [x_l][y][z], `out` = half spectrum [y_l][n2/2+1][x]) and
 * complex-to-real (BACKWARD: the reverse) over the same slabs.  The reference has no R2C; this follows the C2C wrapper above.
 * `in` and `out` are separate buffers of the sizes dfft_local_size_r2c_3d gives, so bufferDev1 / bufferDev2 hold real or
 * complex data according to the direction (bufferDev1 = the input side).  Executed and destroyed like a C2C plan. */
inline fft_mpi_3d_plan_p fft_mpi_plan_dft_r2c_3d(longInt64 n0, longInt64 n1, longInt64 n2, void* in, void* out, MPI_Comm, int devIdx,
                                                 int devCountInNode, int totalDevCount, int direction)
{
    fft_mpi_3d_plan_p plan = new fft_mpi_3d_plan();
    plan->N[0] = (int)n0; plan->N[1] = (int)n1; plan->N[2] = (int)n2;
    plan->direction = direction;
    plan->locGPUIdx = devIdx; plan->devCountInNode = devCountInNode; plan->totalDevCount = totalDevCount;
    plan->globalDevIdx = devIdx;
    plan->isLastDevice = devIdx == totalDevCount - 1;
    plan->inDev = (Complex*)in; plan->outDev = (Complex*)out;
    plan->isInplace = false;
    dfft_comm comm = totalDevCount > 1 ? dfft_shim::local_comm(totalDevCount) : nullptr;
    DFFT_CHECK(dfft_plan_r2c_3d(n0, n1, n2, in, out, comm, devIdx, totalDevCount, direction, DFFT_DOUBLE, DFFT_EXCHANGE_AUTO, &plan->impl));
    DFFT_CHECK(dfft_plan_counts(plan->impl, nullptr, nullptr, &plan->maxDataCountInDevice));
    void *b1 = nullptr, *b2 = nullptr;
    DFFT_CHECK(dfft_plan_buffers(plan->impl, &b1, &b2));
    plan->bufferDev1 = (Complex*)b1; plan->bufferDev2 = (Complex*)b2;
    plan->nodeDataDev = nullptr;
    return plan;
}

/* fft_mpi_3d_api.cpp:181-214: synchronous, prints the stage line on forward */
inline void fft_mpi_execute_dft_3d_c2c(fft_mpi_3d_plan_p p)
{
    DFFT_CHECK(dfft_execute(p->impl));
    DFFT_CHECK(dfft_get_timings(p->impl, p->t));
    if (p->direction == FORWARD)
        printf("t0: %lf, t1: %lf, t2: %lf, t3: %lf, total: %lf\n", p->t[0] * 1e-3, p->t[1] * 1e-3, p->t[2] * 1e-3,
               p->t[3] * 1e-3, p->t[4] * 1e-3);   /* seconds, api.cpp:201 */
}

inline void fft_mpi_destroy_plan(fft_mpi_3d_plan_p plan)
{
    DFFT_CHECK(dfft_destroy(plan->impl));
    delete plan;
}

#endif /* DFFT_FFT_MPI_3D_API_SHIM_H */
