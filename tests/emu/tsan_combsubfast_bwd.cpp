// ThreadSanitizer driver for the emulated CombSubFast backward kernel (built by
// tests/test_emu_combsubfast_backward.py with -fsanitize=thread).  A CUDA shared-memory race (missing / misplaced
// __syncthreads) is a data race between the std::threads of host_emu.h, which TSan reports; tests/test_emu_tsan.py's
// negative control shows that the detector sees through the emulated barrier.
#include <cstdio>
#include <random>
#include <vector>

#include "emu_combsubfast_bwd.cpp"

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    auto fill = [&](std::vector<float>& v, float scale, float shift = 0.f) { for (auto& e : v) e = nd(rng) * scale + shift; };
    const int B = 1, nF = 7, T = nF * 512, C = 3 * 513;
    std::vector<float> comb(B * T), noise(B * T), dense(B * nF * C), g(B * T), grad(B * nF * C);
    fill(comb, 0.3f); fill(noise, 0.5f); fill(dense, 0.3f, -1.f); fill(g, 1.f);
    const float* d = dense.data();
    // explicit noise with 2-row chunks (several CTAs, frames nF-1 and nF paired in the last one), then in-kernel
    // noise in one chunk of an even frame count (frame nF alone in its pair, added to the stored row)
    emu_combsubfast_bwd(comb.data(), d, d + 513, d + 1026, C, noise.data(), 1, 0, g.data(), B, nF, 2, grad.data());
    emu_combsubfast_bwd(comb.data(), d, d + 513, d + 1026, C, nullptr, 1, 0, g.data(), B, nF - 1, 32, grad.data());
    double s = 0;
    for (float v : grad) s += v;
    std::printf("done %g\n", s);
    return 0;
}
