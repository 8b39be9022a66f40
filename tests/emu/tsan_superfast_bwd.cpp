// ThreadSanitizer driver for the emulated CombSubSuperFast backward kernel (built by
// tests/test_emu_superfast_backward.py with -fsanitize=thread).  A CUDA shared-memory race (missing / misplaced
// __syncthreads) is a data race between the std::threads of host_emu.h, which TSan reports; tests/test_emu_tsan.py's
// negative control shows that the detector sees through the emulated barrier.
#include <cstdio>
#include <random>
#include <vector>

#include "emu_superfast_bwd.cpp"

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    auto fill = [&](std::vector<float>& v, float scale, float shift = 0.f) { for (auto& e : v) e = nd(rng) * scale + shift; };
    const int B = 1, nF = 9, T = nF * 512, C = 4 * 1025;
    std::vector<float> par(B * nF * 4), noise(B * T), dense(B * nF * C), g(B * T), grad(B * nF * C);
    for (int k = 0; k < nF; ++k) {
        par[4 * k] = 0.005f + 0.0001f * k;
        par[4 * k + 1] = k + 1 < nF ? 0.0001f : 0.f;
        par[4 * k + 2] = 0.1f * k - (int)(0.1f * k);
        par[4 * k + 3] = 0.f;
    }
    fill(noise, 1.f); fill(dense, 0.3f, -1.f); fill(g, 1.f);
    const float* d = dense.data();
    // explicit noise with 5-hop chunks (several CTAs, the held frame in the last one), then in-kernel noise, one chunk
    emu_superfast_bwd(par.data(), d, d + 1025, d + 2050, d + 3075, C, noise.data(), 1, 0, g.data(), B, nF, 5, grad.data());
    emu_superfast_bwd(par.data(), d, d + 1025, d + 2050, d + 3075, C, nullptr, 1, 0, g.data(), B, nF, 29, grad.data());
    double s = 0;
    for (float v : grad) s += v;
    std::printf("done %g\n", s);
    return 0;
}
