// fp32 instantiations.  Per-length choices come from kbench sweeps (csrc/tools/kbench.cu):
// small CTAs (finer barriers) win for the contiguous pass, 128-byte row segments (C = 8 complex
// doubles) for the strided ones.
#include "dfft_kernels_inst.cuh"
namespace dfft {
void register_f32(std::vector<SizeEntry>& v)
{
    using T = float;
    v.push_back(make_entry<T, Cfg<Sched<4, 2, 2, 2>, 64, false, 4, true>, Cfg<Sched<4, 2, 2, 2>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<8, 4, 4, 2>, 64, false, 4, true>, Cfg<Sched<8, 4, 4, 2>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<16, 4, 4, 4>, 32, false, 4, true>, Cfg<Sched<16, 4, 4, 4>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<32, 8, 8, 4>, 32, false, 4, true>, Cfg<Sched<32, 8, 8, 4>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<64, 8, 8, 8>, 16, true, 4, true>, Cfg<Sched<64, 8, 8, 8>, 16, true, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<128, 16, 16, 8>, 16, false, 4, true>, Cfg<Sched<128, 16, 16, 8>, 16, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<256, 16, 16, 16>, 8, false, 4, true>, Cfg<Sched<256, 16, 16, 16>, 8, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<512, 8, 8, 8, 8>, 2, true, 4, true>, Cfg<Sched<512, 16, 8, 8, 8>, 8, false, 2, false>>());
    // fp32 strided passes want 16 columns (128-byte row segments) and 32 points per thread
    v.push_back(make_entry<T, Cfg<Sched<1024, 16, 16, 8, 8>, 2, false, 4, true>, Cfg<Sched<1024, 32, 16, 16, 4>, 16, false, 1, false>>());
    v.push_back(make_entry<T, Cfg<Sched<2048, 16, 16, 16, 8>, 1, false, 4, false>, Cfg<Sched<2048, 16, 16, 16, 8>, 4, false, 1, false>>());
    v.push_back(make_entry<T, Cfg<Sched<4096, 16, 16, 16, 16>, 1, false, 2, false>, Cfg<Sched<4096, 16, 16, 16, 16>, 2, false, 1, false>>());
    // mixed radix
    v.push_back(make_entry<T, Cfg<Sched<768, 12, 4, 4, 4, 4, 3>, 2, false, 4, true>, Cfg<Sched<768, 24, 8, 8, 4, 3>, 16, false, 1, false>>());
    v.push_back(make_entry<T, Cfg<Sched<384, 12, 4, 4, 4, 3, 2>, 4, false, 4, true>, Cfg<Sched<384, 12, 4, 4, 4, 3, 2>, 8, false, 2, false>>());
    v.push_back(make_entry<T, Cfg<Sched<192, 12, 4, 4, 4, 3>, 8, false, 4, true>, Cfg<Sched<192, 12, 4, 4, 4, 3>, 8, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<96, 12, 4, 4, 3, 2>, 16, false, 4, true>, Cfg<Sched<96, 12, 4, 4, 3, 2>, 16, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<48, 12, 4, 4, 3>, 32, false, 4, true>, Cfg<Sched<48, 12, 4, 4, 3>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<24, 6, 3, 2, 2, 2>, 32, false, 4, true>, Cfg<Sched<24, 6, 3, 2, 2, 2>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<12, 6, 3, 2, 2>, 64, false, 4, true>, Cfg<Sched<12, 6, 3, 2, 2>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<6, 6, 3, 2>, 64, false, 4, true>, Cfg<Sched<6, 6, 3, 2>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<9, 3, 3, 3>, 32, false, 4, true>, Cfg<Sched<9, 3, 3, 3>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<10, 10, 5, 2>, 64, false, 4, true>, Cfg<Sched<10, 10, 5, 2>, 32, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<100, 10, 5, 5, 2, 2>, 16, false, 4, true>, Cfg<Sched<100, 10, 5, 5, 2, 2>, 16, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<125, 5, 5, 5, 5>, 8, false, 4, true>, Cfg<Sched<125, 5, 5, 5, 5>, 8, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<49, 7, 7, 7>, 16, false, 4, true>, Cfg<Sched<49, 7, 7, 7>, 16, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<243, 9, 3, 3, 3, 3, 3>, 8, false, 4, true>, Cfg<Sched<243, 9, 3, 3, 3, 3, 3>, 8, false, 4, true>>());
    v.push_back(make_entry<T, Cfg<Sched<1000, 10, 5, 5, 5, 2, 2, 2>, 2, false, 4, true>, Cfg<Sched<1000, 10, 5, 5, 5, 2, 2, 2>, 4, false, 2, false>>());
}
}  // namespace dfft
