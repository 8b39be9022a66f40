// ThreadSanitizer driver for the emulated reflow sampler kernels (built by tests/test_emu_reflow.py with
// -fsanitize=thread).  They use no shared memory and no barrier; every output element must have exactly one owning
// thread across the grid-stride loop, so two threads writing one element would be a data race that TSan reports.
#include <cstdio>
#include <random>
#include <vector>

#include "emu_reflow.cpp"

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    const int B = 2, T = 13, M = 12, D = 64, LD = 3 * D, N = B * T;
    auto vec = [&](size_t n) { std::vector<float> v(n); for (auto& e : v) e = nd(rng); return v; };
    auto noise = vec((size_t)B * M * T), gt = vec((size_t)N * M), g = vec((size_t)N * D), bias = vec(D), h = vec((size_t)N * D),
         step = vec((size_t)B * LD), cond = vec((size_t)N * LD), gm = vec((size_t)N * M), bm = vec(M), acc = vec((size_t)N * M);
    std::vector<float> x((size_t)N * M), hi((size_t)N * D), lo((size_t)N * D), out((size_t)N * M);
    emu_rf_start(noise.data(), gt.data(), 0.7f, 0.3f, -12.f, 14.f, B, T, M, x.data(), hi.data(), lo.data());
    emu_rf_layer_input(g.data(), bias.data(), h.data(), 0, step.data(), LD, cond.data(), LD, B, T, D, hi.data(), lo.data());
    emu_rf_layer_input(g.data(), bias.data(), h.data(), 1, nullptr, 0, nullptr, 0, B, T, D, hi.data(), nullptr);
    for (int s = 0; s < 4; ++s) emu_rf_ode(gm.data(), bm.data(), x.data(), acc.data(), s, 0.1f, N, M, hi.data(), lo.data());
    emu_rf_ode(gm.data(), bm.data(), x.data(), nullptr, -1, 0.1f, N, M, hi.data(), nullptr);
    emu_rf_finish(x.data(), -12.f, 14.f, N * M, out.data());
    double s = 0;
    for (float v : out) s += v;
    for (float v : h) s += v;
    std::printf("done %g\n", s);
    return 0;
}
