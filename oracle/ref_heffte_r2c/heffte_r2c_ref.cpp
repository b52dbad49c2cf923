// heffte_r2c_ref.cpp -- TEST INFRASTRUCTURE ONLY (oracle/).  A C entry point around the UNMODIFIED heFFTe 2.1.0 of the
// reference tree (heffte/heffteBenchmark, `stock` CPU backend): its real-to-complex transform heffte::fft3d_r2c
// (include/heffte_fft3d_r2c.h), used to anchor the R2C / C2R layout and sign convention of dfft_plan_r2c_3d.
// World arrays are natural order A[x][y][z], z fastest; heFFTe's index 0 is the fastest one, so its boxes are (z, y, x) and
// r2c_direction = 0 is our z axis.  Real boxes are x-slabs, complex boxes y-slabs of the half-spectrum world (z cut to
// n2/2 + 1), as in ../ref_heffte/heffte_ref.cpp for the C2C transform; the ranks are threads behind ../ref_heffte/mpi.h.
#include <algorithm>
#include <complex>
#include <vector>

#include "heffte.h"

namespace {

struct Job {
    int n0, n1, n2, P, direction, scale_full;
    const void* in;
    void* out;
};

template <typename T> void transform_rank(void* vjob)
{
    Job& j = *static_cast<Job*>(vjob);
    using cplx = std::complex<T>;
    MPI_Comm comm = MPI_COMM_WORLD;
    const int me = heffte::mpi::comm_rank(comm);
    const int nzh = j.n2 / 2 + 1;
    heffte::box3d<> const rworld = {{0, 0, 0}, {j.n2 - 1, j.n1 - 1, j.n0 - 1}};
    heffte::box3d<> const cworld = rworld.r2c(0);
    std::vector<heffte::box3d<>> rboxes = heffte::split_world(rworld, {1, 1, j.P});   // x-slabs of the real array
    std::vector<heffte::box3d<>> cboxes = heffte::split_world(cworld, {1, j.P, 1});   // y-slabs of the half spectrum
    heffte::plan_options o = heffte::default_options<heffte::backend::stock>();
    o.use_pencils = false;
    heffte::fft3d_r2c<heffte::backend::stock> fft(rboxes[me], cboxes[me], 0, comm, o);
    const heffte::box3d<>& rb = rboxes[me];
    const heffte::box3d<>& cb = cboxes[me];
    auto ridx = [&](long long x, long long y, long long z) { return ((size_t)x * j.n1 + y) * j.n2 + z; };
    auto cidx = [&](long long x, long long y, long long z) { return ((size_t)x * j.n1 + y) * nzh + z; };
    std::vector<T> r((size_t)fft.size_inbox());
    std::vector<cplx> c((size_t)fft.size_outbox());
    size_t k = 0;
    if (j.direction > 0) {
        const T* win = static_cast<const T*>(j.in);
        for (int x = rb.low[2]; x <= rb.high[2]; x++)
            for (int y = rb.low[1]; y <= rb.high[1]; y++)
                for (int z = rb.low[0]; z <= rb.high[0]; z++) r[k++] = win[ridx(x, y, z)];
        fft.forward(r.data(), c.data());
        cplx* wout = static_cast<cplx*>(j.out);
        k = 0;
        for (int x = cb.low[2]; x <= cb.high[2]; x++)
            for (int y = cb.low[1]; y <= cb.high[1]; y++)
                for (int z = cb.low[0]; z <= cb.high[0]; z++) wout[cidx(x, y, z)] = c[k++];
    } else {
        const cplx* win = static_cast<const cplx*>(j.in);
        for (int x = cb.low[2]; x <= cb.high[2]; x++)
            for (int y = cb.low[1]; y <= cb.high[1]; y++)
                for (int z = cb.low[0]; z <= cb.high[0]; z++) c[k++] = win[cidx(x, y, z)];
        fft.backward(c.data(), r.data(), j.scale_full ? heffte::scale::full : heffte::scale::none);
        T* wout = static_cast<T*>(j.out);
        k = 0;
        for (int x = rb.low[2]; x <= rb.high[2]; x++)
            for (int y = rb.low[1]; y <= rb.high[1]; y++)
                for (int z = rb.low[0]; z <= rb.high[0]; z++) wout[ridx(x, y, z)] = r[k++];
    }
}

}  // namespace

extern "C" {

/* world-array R2C / C2R by the reference library over P slab ranks.  direction +1: in = real A[x][y][z] (n0*n1*n2),
 * out = half spectrum [x][y][n2/2+1] (e^{-i...}, unnormalised); direction -1: the reverse, unnormalised unless scale_full.
 * precision 0 = double, 1 = float.  Returns 0, -1 when P does not fit the boxes, -2 on an exception. */
int heffte_ref_fft3d_r2c(int n0, int n1, int n2, int P, const void* in, void* out, int direction, int precision, int scale_full)
{
    if (P < 1 || P > n0 || P > n1 || n0 < 1 || n1 < 1 || n2 < 1) return -1;
    Job j{n0, n1, n2, P, direction, scale_full, in, out};
    try {
        if (precision == 0) tmpi_run(P, transform_rank<double>, &j);
        else tmpi_run(P, transform_rank<float>, &j);
    } catch (...) { return -2; }
    return 0;
}
}
