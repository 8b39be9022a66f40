// CPU execution of csrc/hifigan.cu's kernel source (see host_emu.h).  Built by tests/test_emu_hifigan.py; the same
// test builds it with -DEMU_ASAN under AddressSanitizer (main below) and tsan_main.cpp includes it for ThreadSanitizer.
// emu_hg_conv runs the <BM, BN> instantiation it is given, not the one hifigan_conv_launch would pick.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#define gridDim (emu::grid_dim)
#define blockDim (emu::block_dim)
#include "../../ddsp_svc_b200/csrc/hifigan.cu"

namespace {
alignas(16) float smem[1 << 16];          // hg_conv_kernel's `extern __shared__` array
alignas(16) float sw[1 << 14];            // hg_post_kernel's

template <int BM, int BN>
int run_conv(const HgConvParams& p) {
    const int halo = p.dil * (p.k - 1) / 2;
    if ((size_t)3 * (BM + 2 * halo) * kKS > sizeof smem / sizeof(float) || p.N % BN || p.Cin % kKC) return -2;
    emu::shared_window(smem, sizeof smem);
    emu::launch(dim3{(unsigned)((p.T + BM - 1) / BM), (unsigned)(p.N / BN), (unsigned)p.B}, kWarps * 32,
                [&] { hg_conv_kernel<BM, BN>(p); });
    return 0;
}
}  // namespace

extern "C" int emu_hg_conv(int BM, int BN, const float* x, long long sb, long long st, long long sc, int B, int T,
                           int Cin, const float* w, const float* bias, int k, int dil, int N, int lrelu,
                           const float* residual, const float* accum, float div, int up, const float* src,
                           const float* wn, const float* bn, int n_k, int n_stride, int n_pad, float* out) {
    HgConvParams p{x, sb, st, sc, B, T, Cin, w, bias, k, dil, N, lrelu, residual, accum, div, up, src, wn, bn,
                   n_k, n_stride, n_pad, out};
    if (BM == 64 && BN == 32) return run_conv<64, 32>(p);
    if (BM == 64 && BN == 16) return run_conv<64, 16>(p);
    if (BM == 128 && BN == 32) return run_conv<128, 32>(p);
    if (BM == 128 && BN == 16) return run_conv<128, 16>(p);
    return -1;
}

extern "C" int emu_hg_post(const float* x, const float* w, const float* bias, int B, int T, int C, int ctas,
                           int threads, float* out) {
    if ((size_t)7 * C > sizeof sw / sizeof(float)) return -2;
    emu::launch((unsigned)ctas, 1u, (unsigned)threads, [&] { hg_post_kernel(x, w, bias, B, T, C, out); });
    return 0;
}

#ifdef EMU_ASAN
// Every input in a heap buffer of exactly its logical size, at the edge shapes: any read or write past a tensor is an
// AddressSanitizer report.  Values are arbitrary (the numerics are tests/test_emu_hifigan.py's business).
#include <random>
#include <vector>
int main() {
    std::mt19937 rng(3);
    std::uniform_real_distribution<float> ud(-1.f, 1.f);
    auto vec = [&](size_t n) { std::vector<float> v(n); for (auto& e : v) e = ud(rng); return v; };
    int rc = 0;
    for (int BM : {64, 128})
        for (int BN : {16, 32})
            for (int T : {1, BM + 1}) {
                const int B = 2, C = 32, k = 7, d = 3;
                auto x = vec((size_t)B * T * C), w = vec((size_t)2 * k * C * C), b = vec(C), r = vec((size_t)B * T * C),
                     a = vec((size_t)B * T * C), o = vec((size_t)B * T * C);
                rc |= emu_hg_conv(BM, BN, x.data(), (long long)T * C, C, 1, B, T, C, w.data(), b.data(), k, d, C, 1,
                                  r.data(), a.data(), 3.f, 0, nullptr, nullptr, nullptr, 0, 0, 0, o.data());
                auto xc = vec((size_t)B * C * T);                                   // channel-major conv_pre input
                rc |= emu_hg_conv(BM, BN, xc.data(), (long long)C * T, 1, T, B, T, C, w.data(), b.data(), k, 1, C, 0,
                                  nullptr, nullptr, 1.f, 0, nullptr, nullptr, nullptr, 0, 0, 0, o.data());
                const int u = 2, Co = 16, s = 4, nk = 8;                            // transposed stage with its source
                auto wt = vec((size_t)2 * 3 * C * u * Co), bt = vec(Co), src = vec((size_t)B * T * u * s),
                     wn = vec((size_t)Co * nk), bn = vec(Co), ot = vec((size_t)B * T * u * Co);
                rc |= emu_hg_conv(BM, 16, x.data(), (long long)T * C, C, 1, B, T, C, wt.data(), bt.data(), 3, 1, u * Co,
                                  1, nullptr, nullptr, 1.f, u, src.data(), wn.data(), bn.data(), nk, s, s / 2,
                                  ot.data());
            }
    for (int T : {1, 2, 5}) {
        const int B = 3, C = 16;
        auto x = vec((size_t)B * T * C), w = vec(7 * C), b = vec(1), o = vec((size_t)B * T);
        rc |= emu_hg_post(x.data(), w.data(), b.data(), B, T, C, 2, 32, o.data());
    }
    std::printf("done %d\n", rc);
    return rc;
}
#endif
