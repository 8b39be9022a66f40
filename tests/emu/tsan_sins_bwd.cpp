// ThreadSanitizer driver for the emulated Sins backward kernels (built by tests/test_emu_sins_backward.py with
// -fsanitize=thread).  A CUDA shared-memory race (missing / misplaced __syncthreads) is a data race between the
// std::threads of host_emu.h, which TSan reports; tests/test_emu_tsan.py's negative control shows that the detector
// sees through the emulated barrier.
#include <cstdio>
#include <random>
#include <vector>

#include "emu_sins_bwd.cpp"

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    auto fill = [&](std::vector<float>& v, float scale, float shift = 0.f) { for (auto& e : v) e = nd(rng) * scale + shift; };
    const int B = 1, nF = 3, T = nF * 512;
    double sum = 0;
    // (H, Ma, Mn): one harmonic group with equal filters, two groups with unequal ones
    const int shapes[2][3] = {{40, 65, 65}, {200, 33, 129}};
    for (const auto& sh : shapes) {
        const int H = sh[0], Ma = sh[1], Mn = sh[2], C = H + Ma + Mn, La = 2 * (Ma - 1), Ln = 2 * (Mn - 1);
        std::vector<float> f0(B * nF), dense(B * nF * C), sinus(B * T), noise(B * T), irA(B * nF * La), irN(B * nF * Ln),
            g(B * T), gh(B * T), gn(B * T), dx(B * T), grad(B * nF * C);
        std::vector<double> fph(B * nF);
        for (int k = 0; k < nF; ++k) { f0[k] = 150.f + 10.f * k; fph[k] = 0.37 * k; }
        fill(dense, 0.3f, -1.f); fill(sinus, 0.1f); fill(noise, 0.5f); fill(irA, 0.1f); fill(irN, 0.01f);
        fill(g, 1.f); fill(gh, 1.f); fill(gn, 1.f);
        const float* d = dense.data();
        emu_sins_bwd(f0.data(), fph.data(), d, d + H, d + H + Ma, C, sinus.data(), irA.data(), irN.data(), noise.data(),
                     1, 0, g.data(), gh.data(), gn.data(), B, nF, H, Ma, Mn, 44100.0, dx.data(), grad.data());
        emu_sins_bwd(f0.data(), fph.data(), d, d + H, d + H + Ma, C, sinus.data(), irA.data(), irN.data(), nullptr,
                     1, 0, g.data(), nullptr, nullptr, B, nF, H, Ma, Mn, 44100.0, dx.data(), grad.data());
        for (float v : grad) sum += v;
    }
    std::printf("done %g\n", sum);
    return 0;
}
