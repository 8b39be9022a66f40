// ThreadSanitizer driver for the emulated mel backward kernel (built by tests/test_emu_mel_backward.py with
// -fsanitize=thread).  A CUDA shared-memory race (missing / misplaced __syncthreads) is a data race between the
// std::threads of host_emu.h, which TSan reports; tests/test_emu_tsan.py's negative control shows that the detector sees
// through the emulated barrier.
#include <cstdio>
#include <random>
#include <vector>

#include "emu_mel_bwd.cpp"

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    const int n_mels = 16, hop = 512, T = 4 * 512 + 77;
    std::vector<float> y(T), window(kN), basis((size_t)n_mels * kBins, 0.f), dy(T);
    std::vector<int> lohi(2 * n_mels), bins(2 * kBins, 0);
    for (auto& v : y) v = nd(rng);
    for (int n = 0; n < kN; ++n) window[n] = 0.5f - 0.5f * std::cos(2.0 * M_PI * n / kN);
    for (int m = 0; m < n_mels; ++m) {              // overlapping triangles of 40 bins
        lohi[2 * m] = 20 * m; lohi[2 * m + 1] = 20 * m + 40;
        for (int k = 20 * m; k < 20 * m + 40; ++k) basis[(size_t)m * kBins + k] = 0.05f * (1 + (k < 20 * m + 20 ? k - 20 * m : 20 * m + 40 - k));
    }
    for (int k = 0; k < kBins; ++k) {
        int lo = -1, hi = 0;
        for (int m = 0; m < n_mels; ++m) if (basis[(size_t)m * kBins + k] != 0.f) { if (lo < 0) lo = m; hi = m + 1; }
        bins[2 * k] = lo < 0 ? 0 : lo; bins[2 * k + 1] = hi;
    }
    const int nF = b2d_mel_frames(T, kN, kN, hop);
    std::vector<float> g((size_t)n_mels * nF);
    for (auto& v : g) v = nd(rng);
    // two chunks (halo frames and both reflected ends), then one chunk holding the whole utterance
    emu_mel_bwd(y.data(), window.data(), basis.data(), lohi.data(), bins.data(), g.data(), 0, nF, 1, 1, T, hop, n_mels,
                1e-5f, 2 * hop, dy.data());
    emu_mel_bwd(y.data(), window.data(), basis.data(), lohi.data(), bins.data(), g.data(), 0, nF, 1, 1, T, hop, n_mels,
                1e-5f, 8192, dy.data());
    double s = 0;
    for (float v : dy) s += v;
    std::printf("done %g\n", s);
    return 0;
}
