// batchFFT -- single-GPU batched 1-D / 2-D / 3-D C2C benchmark with the argv, stdout lines and CSV columns of the
// reference's templateFFT/batchTest/Test_1D.cpp and Test_2D.cpp (the only kernel-level numbers the reference
// publishes: templateFFT/csv/batch_result1D.csv, batch_result2D.csv):
//     batchFFT 1d X Y Z num_iter printResult [csv]      Y is overridden to 2^26 / X     (Test_1D.cpp:208-212)
//     batchFFT 2d X Y Z num_iter printResult [csv]      Z is overridden to 2^26 / (X*Y) (Test_2D.cpp:205)
//     batchFFT 3d X Y Z num_iter printResult [csv]      batch = 2^26 / (X*Y*Z) volumes (the reference's FFTdim = 3 application)
// Forward on the ramp input i+1, timing loop of num_iter forward launches (events on the plan's stream), inverse,
// round-trip max error -- through the lines-plan API of libdfft.so (initializeFFT / launchFFTKernel / deleteFFT).
#include <cuda_runtime.h>

#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>

#include "dfft.h"

#define CK(stmt)                                                                                      \
    do {                                                                                              \
        int rc_ = (int)(stmt);                                                                        \
        if (rc_ != 0) {                                                                               \
            fprintf(stderr, "[%s:%d] '%s' failed with %d: %s\n", __FILE__, __LINE__, #stmt, rc_, dfft_last_error()); \
            exit(EXIT_FAILURE);                                                                       \
        }                                                                                             \
    } while (0)

int main(int argc, char* argv[])
{
    if (argc < 7 || (strcmp(argv[1], "1d") && strcmp(argv[1], "2d") && strcmp(argv[1], "3d"))) {
        printf("usage: batchFFT 1d|2d|3d X Y Z num_iter printResult [csv_file]\n");
        return EXIT_FAILURE;
    }
    const bool two = !strcmp(argv[1], "2d"), three = !strcmp(argv[1], "3d");
    long long X = atoll(argv[2]), Y = atoll(argv[3]), Z = atoll(argv[4]);
    const int num_iter = atoi(argv[5]), printResult = atoi(argv[6]);
    const char* csv = argc > 7 ? argv[7] : nullptr;
    const long long total = 64LL * 32 * 32768;   // 2^26 complex doubles = 1 GiB
    if (X < 1 || num_iter < 1) { printf("bad arguments\n"); return EXIT_FAILURE; }
    long long B = 1;   // 3-D: volumes per batch
    if (three) { if (Y < 1 || Z < 1 || X * Y * Z > total) { printf("size too large for the 2^26-element buffer\n"); return EXIT_FAILURE; } B = total / (X * Y * Z); }
    else if (two) { if (Y < 1) return EXIT_FAILURE; Z = total / (X * Y); }
    else { Y = total / X; Z = 1; }
    if (Y < 1 || Z < 1) { printf("size too large for the 2^26-element buffer\n"); return EXIT_FAILURE; }
    const long long N = X * Y * Z * B;
    printf("1 - FFT + iFFT C2C %s in double precision LUT\n", three ? "3D" : (two ? "2D" : "1D"));

    double* in = (double*)malloc(sizeof(double) * 2 * N);
    double* out = (double*)malloc(sizeof(double) * 2 * N);
    for (long long i = 0; i < N; i++) { in[2 * i] = (double)((int)i) + 1.0; in[2 * i + 1] = 0.0; }   // Test_1D.cpp:49-52
    const size_t bytes = sizeof(double) * 2 * (size_t)N;
    void *buf = nullptr, *tmp = nullptr;
    CK(cudaMalloc(&buf, bytes));
    CK(cudaMalloc(&tmp, bytes));
    CK(cudaMemcpy(buf, in, bytes, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(tmp, in, bytes, cudaMemcpyHostToDevice));

    dfft_lines_plan plan = nullptr;
    if (three) CK(dfft_lines_plan_create_3d((int)X, (int)Y, (int)Z, B, DFFT_DOUBLE, &plan));
    else if (two) CK(dfft_lines_plan_create_2d((int)X, (int)Y, Z, DFFT_DOUBLE, &plan));
    else CK(dfft_lines_plan_create((int)X, 1, Y, Y, X, 0, DFFT_DOUBLE, &plan));
    cudaStream_t st = (cudaStream_t)dfft_lines_stream(plan);

    CK(dfft_lines_execute(plan, buf, DFFT_FORWARD));
    CK(dfft_lines_synchronize(plan));
    CK(cudaMemcpy(out, buf, bytes, cudaMemcpyDeviceToHost));

    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(dfft_lines_execute(plan, tmp, DFFT_FORWARD));   // warm-up
    CK(cudaEventRecord(e0, st));
    for (int i = 0; i < num_iter; i++) CK(dfft_lines_execute(plan, tmp, DFFT_FORWARD));
    CK(cudaEventRecord(e1, st));
    CK(cudaEventSynchronize(e1));
    float elapsed = 0.f;
    CK(cudaEventElapsedTime(&elapsed, e0, e1));
    const double avg = elapsed / num_iter;
    const double opscount = three ? 5.0 * (double)N * std::log((double)(X * Y * Z)) / std::log(2.0)
                          : two ? 5.0 * (double)N * std::log((double)(X * Y)) / std::log(2.0)
                                : (double)Y * 5.0 * (double)X * std::log((double)X) / std::log(2.0);
    if (three)
        printf("FFT: %lldx%lldx%lldx%lld Buffer: %f MB avg_hip_time: %0.6f ms Gflops: %0.6f num_iter: %d \n", X, Y, Z, B, bytes / 1024.0 / 1024.0, avg,
               opscount / (1e6 * avg), num_iter);
    else
        printf("FFT: %lldx%lldx%lld Buffer: %f MB avg_hip_time: %0.6f ms Gflops: %0.6f num_iter: %d \n", X, Y, Z, bytes / 1024.0 / 1024.0, avg,
               opscount / (1e6 * avg), num_iter);

    CK(dfft_lines_execute(plan, buf, DFFT_BACKWARD));
    CK(dfft_lines_synchronize(plan));
    CK(cudaMemcpy(out, buf, bytes, cudaMemcpyDeviceToHost));
    if (printResult == 1) {
        for (long long i = 0; i < 8 && i < N; i++)
            std::cout << "element " << i << " input:  (" << in[2 * i] << "," << in[2 * i + 1] << ") output: (" << out[2 * i] << "," << out[2 * i + 1] << ")" << std::endl;
        for (long long i = (N > 8 ? N - 8 : 0); i < N; i++)
            std::cout << "element " << i << " input:  (" << in[2 * i] << "," << in[2 * i + 1] << ") output: (" << out[2 * i] << "," << out[2 * i + 1] << ")" << std::endl;
    }
    const double norm = three ? (double)(X * Y * Z) : (two ? (double)(X * Y) : (double)X);
    double maxErr = 0.0;
    for (long long i = 0; i < N; i++) {   // Test_1D.cpp:169-175
        double t1 = in[2 * i] - out[2 * i] / norm, t2 = in[2 * i + 1] - out[2 * i + 1] / norm;
        double t3 = std::sqrt(t1 * t1 + t2 * t2);
        maxErr = maxErr >= t3 ? maxErr : t3;
    }
    std::cout << "Max error: " << maxErr << std::endl;
    if (csv) {   // columns of runTest1D_opt.sh:4 : X,Y,Z,Buffer,hip_time,GFlops,num_iter,bandwidth,max error
        // one read + one write per axis (Test_1D.cpp:181, Test_2D.cpp:180), whether or not two axes share one sweep
        const double transfers = three ? 6.0 : (two ? 4.0 : 2.0);
        std::ofstream f(csv, std::ios::app);
        f << X << ',' << Y << ',' << Z << ',' << bytes / 1024.0 / 1024.0 << ',' << avg << ',' << opscount / (1e6 * avg) << ',' << num_iter << ','
          << bytes / 1024.0 / 1024.0 / 1.024 * transfers / avg << ',' << maxErr << std::endl;
    }
    CK(dfft_lines_destroy(plan));
    cudaFree(buf); cudaFree(tmp);
    free(in); free(out);
    return 0;
}
