// ThreadSanitizer driver for the emulated RSS loss kernels (built by tests/test_emu_rss_loss.py with
// -fsanitize=thread).  A CUDA shared-memory race (missing / misplaced __syncthreads) is a data race between the
// std::threads of host_emu.h, which TSan reports.  One scale per transform size; the tables are built here in float64
// the way ddsp_svc_b200.loss.table_host builds them (naive DFT: the sizes are small).
#include <complex>
#include <cstdio>
#include <random>
#include <vector>

#include "emu_rss_loss.cpp"

static std::vector<float> make_table(int n) {
    const int M = bluestein_size(n);
    std::vector<float> t(b2d_rss_table_floats(n), 0.f);
    double ss = 0;
    for (int m = 0; m < n; ++m) {
        const float w = (float)(0.5 - 0.5 * std::cos(2.0 * M_PI * m / n));
        t[kWinOff + m] = w;
        ss += (double)w * w;
    }
    t[0] = (float)std::sqrt(ss);
    std::vector<std::complex<double>> c(n), h(M);
    for (long long m = 0; m < n; ++m) {
        c[m] = std::polar(1.0, M_PI * (double)((m * m) % (2LL * n)) / n);
        t[chirp_off(n) + 2 * m] = (float)c[m].real();
        t[chirp_off(n) + 2 * m + 1] = (float)c[m].imag();
        h[m] = c[m];
        if (m) h[M - m] = c[m];
    }
    for (int k = 0; k < M; ++k) {
        std::complex<double> s = 0;
        for (int j = 0; j < M; ++j) s += h[j] * std::polar(1.0, -2.0 * M_PI * (double)((long long)j * k % M) / M);
        s /= M;
        t[hspec_off(n) + 2 * k] = (float)s.real();
        t[hspec_off(n) + 2 * k + 1] = (float)s.imag();
    }
    return t;
}

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    const int B = 1, T = 2 * 1031 + 77;
    const int n_ffts[3] = {300, 1031, 513};
    std::vector<float> xp(T), xt(T), dx(T);
    for (int i = 0; i < T; ++i) { xt[i] = nd(rng); xp[i] = 0.7f * xt[i] + 0.3f * nd(rng); }
    std::vector<std::vector<float>> tabs;
    std::vector<const float*> ptrs;
    for (int n : n_ffts) tabs.push_back(make_table(n));
    for (auto& t : tabs) ptrs.push_back(t.data());
    std::vector<double> part(emu_rss_workspace_doubles(B, T, 3, n_ffts)), norms(3 * B * 2);
    float loss = 0.f, gl = 1.f;
    emu_rss_forward(xp.data(), xt.data(), B, T, 3, n_ffts, ptrs.data(), 1.f, 1e-7f, part.data(), norms.data(), &loss);
    emu_rss_backward(xp.data(), xt.data(), B, T, 3, n_ffts, ptrs.data(), 1.f, 1e-7f, norms.data(), &gl, dx.data());
    double s = 0;
    for (float v : dx) s += v;
    std::printf("done %g %g\n", loss, s);
    return 0;
}
