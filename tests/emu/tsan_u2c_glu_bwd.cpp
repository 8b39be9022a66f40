// ThreadSanitizer driver for the emulated GLU -> depthwise conv -> SiLU backward kernel (built by
// tests/test_emu_u2c_backward.py with -fsanitize=thread).  The kernel has no barrier because every thread keeps to its
// own column of the shared arrays; a thread that strayed into another's column would be a data race between the
// std::threads of host_emu.h, which TSan reports (tests/test_emu_tsan.py's negative control shows the detector works).
#include <cstdio>
#include <random>
#include <vector>

#include "emu_u2c_glu_bwd.cpp"

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    const int B = 2, T = 70, Ci = 128;                     // two tiles per utterance: the halo crosses the tile boundary
    std::vector<float> h((size_t)B * T * 2 * Ci), w((size_t)Ci * kDwK), bias(Ci), gout((size_t)B * T * Ci), gh(h.size()),
        dwb((size_t)Ci * kDwbStride);
    for (auto* v : {&h, &w, &bias, &gout})
        for (auto& x : *v) x = 0.3f * nd(rng);
    if (emu_u2c_glu_bwd(h.data(), w.data(), bias.data(), gout.data(), gh.data(), dwb.data(), B, T, Ci)) return 1;
    double s = 0;
    for (float v : gh) s += v;
    for (float v : dwb) s += v;
    std::printf("done %g\n", s);
    return 0;
}
