// ThreadSanitizer driver for the emulated diffusion sampler kernels (built by tests/test_emu_diffusion.py with
// -fsanitize=thread).  They use no shared memory and no barrier; every output element must have exactly one writing
// thread across the grid-stride loop -- the convolution operand is scattered from each token into its neighbours' rows,
// so two threads writing one element would be a data race that TSan reports.
#include <cstdio>
#include <random>
#include <vector>

#include "emu_diffusion.cpp"

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    const int B = 3, T = 5, C = 8, M = 12, N = B * T, L = 2;
    auto vec = [&](size_t n) { std::vector<float> v(n); for (auto& e : v) e = nd(rng); return v; };
    auto g = vec((size_t)N * 2 * C), bias = vec(2 * C), h = vec((size_t)N * C), skip = vec((size_t)N * C),
         step = vec((size_t)L * C), cond = vec((size_t)N * L * 2 * C), gm = vec((size_t)N * M), bm = vec(M),
         x = vec((size_t)N * M), h1 = vec((size_t)N * M), h2 = vec((size_t)N * M), h3 = vec((size_t)N * M),
         noise = vec((size_t)N * M);
    std::vector<float> coef = {0.5f, -0.25f, 1.1f, 0.3f, 0.2f, -0.1f, 0.05f, 0.7f};
    std::vector<float> hi((size_t)N * 3 * C), lo((size_t)N * 3 * C);
    emu_df_layer(g.data(), bias.data(), h.data(), nullptr, 0, step.data(), 0, 1.f, B, T, C, hi.data(), lo.data());
    emu_df_layer(g.data(), bias.data(), h.data(), skip.data(), 1, step.data() + C, 0, 1.f, B, T, C, hi.data(), lo.data());
    emu_df_layer(g.data(), bias.data(), h.data(), skip.data(), 2, nullptr, 0, 1.41421356f, B, T, C, hi.data(), nullptr);
    emu_df_gate(g.data(), cond.data() + 2 * C, L * 2 * C, N, C, hi.data(), lo.data());
    emu_df_relu(g.data(), bias.data(), N, C, hi.data(), nullptr);
    emu_df_update(gm.data(), bm.data(), coef.data(), x.data(), h3.data(), h1.data(), h2.data(), h3.data(), noise.data(), B, T,
                  M, x.data(), hi.data(), lo.data());
    double s = 0;
    for (float v : x) s += v;
    for (float v : h) s += v;
    for (float v : hi) s += v;
    std::printf("done %g\n", s);
    return 0;
}
