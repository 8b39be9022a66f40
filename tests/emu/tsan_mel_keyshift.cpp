// ThreadSanitizer driver for the emulated keyshift mel kernel (built by tests/test_keyshift_mel.py with
// -fsanitize=thread).  A CUDA shared-memory race (missing / misplaced __syncthreads) is a data race between the
// std::threads of host_emu.h, which TSan reports.  One transform length per instantiation the library launches
// (M = 1024 / 2048 / 4096, with and without the zero-upper first pass); the tables need not be exact for a race check.
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include "emu_mel_keyshift.cpp"

int main() {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    const int n_mels = 16, hop = 256, T = 3 * 256 + 77;
    std::vector<float> y(T), basis((size_t)n_mels * kBins, 0.f);
    std::vector<int> lohi(2 * n_mels);
    for (auto& v : y) v = nd(rng);
    for (int m = 0; m < n_mels; ++m) {
        lohi[2 * m] = 20 * m; lohi[2 * m + 1] = 20 * m + 40;
        for (int k = 20 * m; k < 20 * m + 40; ++k) basis[(size_t)m * kBins + k] = 0.01f;
    }
    double s = 0;
    for (int n : {300, 600, 1000, 1300, 1534, 2731}) {             // (M, ZU): 1024 y/n, 2048 y/n, 4096 y/n
        std::vector<float> table(b2d_mel_keyshift_table_floats(n));
        for (size_t i = 0; i < table.size(); ++i) table[i] = std::cos(0.001f * (float)i);
        const int nF = emu_mel_keyshift_frames(T, n, hop);
        std::vector<float> out((size_t)n_mels * nF);
        emu_mel_keyshift(y.data(), table.data(), basis.data(), lohi.data(), 1, T, n, hop, n_mels, 1e-5f, out.data());
        for (float v : out) s += v;
    }
    std::printf("done %g\n", s);
    return 0;
}
