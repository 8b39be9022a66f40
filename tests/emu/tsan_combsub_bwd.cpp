// ThreadSanitizer driver for the emulated CombSub backward kernels (built by tests/test_emu_combsub_backward.py with
// -fsanitize=thread).  A CUDA shared-memory race (missing / misplaced __syncthreads) is a data race between the
// std::threads of host_emu.h, which TSan reports.
#include <cstdio>
#include <random>
#include <vector>

#include "emu_combsub_bwd.cpp"

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    auto fill = [&](std::vector<float>& v, float scale, float shift = 0.f) { for (auto& e : v) e = nd(rng) * scale + shift; };
    const int B = 1, nF = 3, T = nF * 512;
    double sum = 0;
    // (Ma, Mh, Mn): small filters, and a 1024-tap harmonic filter
    const int shapes[2][3] = {{33, 65, 17}, {9, 513, 5}};
    for (const auto& sh : shapes) {
        const int Ma = sh[0], Mh = sh[1], Mn = sh[2], C = Ma + Mh + Mn, Lh = 2 * (Mh - 1);
        std::vector<float> f0(B * nF), dense(B * nF * C), comb(B * T), allp(B * T), noise(B * T), irH(B * nF * Lh),
            g(B * T), gh(B * T), gn(B * T), da(B * T), grad(B * nF * C);
        for (int k = 0; k < nF; ++k) f0[k] = 150.f + 10.f * k;
        fill(dense, 0.3f, -1.f); fill(comb, 0.1f); fill(allp, 0.1f); fill(noise, 0.5f); fill(irH, 0.1f);
        fill(g, 1.f); fill(gh, 1.f); fill(gn, 1.f);
        const float* d = dense.data();
        emu_combsub_bwd(f0.data(), d, d + Ma, d + Ma + Mh, C, comb.data(), allp.data(), irH.data(), noise.data(), 1, 0,
                        g.data(), gh.data(), gn.data(), B, nF, Ma, Mh, Mn, 44100.0, da.data(), grad.data());
        emu_combsub_bwd(f0.data(), d, d + Ma, d + Ma + Mh, C, comb.data(), allp.data(), irH.data(), nullptr, 1, 0,
                        g.data(), nullptr, nullptr, B, nF, Ma, Mh, Mn, 44100.0, da.data(), grad.data());
        for (float v : grad) sum += v;
    }
    std::printf("done %g\n", sum);
    return 0;
}
