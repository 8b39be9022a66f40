// CPU execution of csrc/rmvpe.cu's kernel source (see host_emu.h).  Built by tests/test_emu_rmvpe.py; the same test
// builds it with -DEMU_ASAN under AddressSanitizer (main below) and tsan_main.cpp includes it for ThreadSanitizer.
// emu_rv_conv runs the <BM, BN> instantiation it is given, with the tile shape launch_conv derives for it.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#define gridDim (emu::grid_dim)
#define blockDim (emu::block_dim)
#include "../../ddsp_svc_b200/csrc/rmvpe.cu"

namespace {
alignas(16) float smem[1 << 16];          // rv_conv_kernel's `extern __shared__` array
alignas(16) float sw[1 << 14];            // rv_conv_small_kernel's
alignas(16) unsigned char smem_raw[kMelSmem];   // rv_mel_kernel's

template <int BM, int BN>
int run_conv(RvConvParams p) {
    p.tF = p.F < BM / 4 ? p.F : BM / 4;
    p.tT = BM / p.tF;
    const int hal = (p.k == 3) + (p.k >= 2);
    if ((size_t)3 * (p.tT + hal) * (p.tF + hal) * kKS > sizeof smem / sizeof(float) || p.N % BN || p.Cin % kKC ||
        BM % p.tF)
        return -2;
    emu::shared_window(smem, sizeof smem);
    emu::launch(dim3{(unsigned)(((p.T + p.tT - 1) / p.tT) * (p.F / p.tF)), (unsigned)(p.N / BN), (unsigned)p.B},
                kWarps * 32, [&] { rv_conv_kernel<BM, BN>(p); });
    return 0;
}
}  // namespace

extern "C" int emu_rv_conv(int BM, int BN, const float* x, int ldx, int B, int T, int F, int Cin, const float* w,
                           const float* bias, int k, int N, int n_valid, int act, int up, const float* res, int ldr,
                           float* out, int ldo) {
    RvConvParams p{x, ldx, B, T, F, Cin, w, bias, k, N, n_valid, act, up, res, ldr, out, ldo, 0, 0};
    if (BM == 64 && BN == 32) return run_conv<64, 32>(p);
    if (BM == 64 && BN == 16) return run_conv<64, 16>(p);
    if (BM == 128 && BN == 32) return run_conv<128, 32>(p);
    if (BM == 128 && BN == 16) return run_conv<128, 16>(p);
    return -1;
}

extern "C" int emu_rv_conv_small(const float* x, long long sb, long long st, long long sf, long long sc, int B, int T,
                                 int F, int Cin, const float* in_scale, const float* in_shift, const float* w,
                                 const float* bias, int k, int Cout, int act, int head, float* out, int ldo) {
    RvSmallParams p{x, sb, st, sf, sc, B, T, F, Cin, in_scale, in_shift, w, bias, k, Cout, act, head, out, ldo};
    if ((size_t)Cout * Cin * k * k > sizeof sw / sizeof(float) || Cout > kSmallMaxCout) return -2;
    emu::launch(3u, 1u, 64u, [&] { rv_conv_small_kernel(p); });           // a grid-stride loop over a short grid
    return 0;
}

extern "C" int emu_rv_pool(const float* x, int ldx, int B, int T, int F, int C, float* out) {
    emu::launch(3u, 1u, 64u, [&] { rv_pool_kernel(x, ldx, B, T, F, C, out); });
    return 0;
}

extern "C" int emu_rv_gru(const float* xg, const float* whh, const float* bhh, int B, int T, float* out) {
    emu::launch(dim3{2 * kGruCta, (unsigned)((B + kGruB - 1) / kGruB), 1}, kGruThreads,
                [&] { rv_gru_kernel(xg, whh, bhh, B, T, out); }, kGruCta);
    return 0;
}

extern "C" int emu_rv_decode(const float* sal, int B, int t_pad, int n_frames, float thred, float* f0) {
    emu::launch(2u, 1u, 64u, [&] { rv_decode_kernel(sal, B, t_pad, n_frames, thred, f0); });
    return 0;
}

extern "C" int emu_rv_resample(const float* x, int B, int N, const float* table, int nw, int orig, int taps, int width,
                               int n_out, float* out) {
    emu::launch(3u, 1u, 64u, [&] { rv_resample_kernel(x, B, N, table, nw, orig, taps, width, n_out, out); });
    return 0;
}

extern "C" int emu_rv_mel(const float* y, int B, int N, const float* window, const float* basis, const int* lohi, int hop,
                          int n_frames, int t_pad, float* out) {
    const RvMelParams p{y, window, basis, lohi, out, N, hop, n_frames, t_pad};
    emu::launch((unsigned)((t_pad + kMelFrames - 1) / kMelFrames), (unsigned)B, b2d_fft_smem::kThreads,
                [&] { rv_mel_kernel(p); });
    return 0;
}

#ifdef EMU_ASAN
// Every input in a heap buffer of exactly its logical size, at the edge shapes: any read or write past a tensor is an
// AddressSanitizer report.  Values are arbitrary (the numerics are tests/test_emu_rmvpe.py's business).
#include <random>
#include <vector>
int main() {
    std::mt19937 rng(5);
    std::uniform_real_distribution<float> ud(-1.f, 1.f);
    auto vec = [&](size_t n) { std::vector<float> v(n); for (auto& e : v) e = ud(rng); return v; };
    int rc = 0;
    for (int BM : {64, 128})
        for (int F : {4, BM / 4})
            for (int k : {1, 3}) {
                const int B = 2, T = 7, C = 16, N = 32;
                auto x = vec((size_t)B * T * F * C), w = vec((size_t)2 * k * k * C * N), b = vec(N),
                     r = vec((size_t)B * T * F * N), o = vec((size_t)B * T * F * N);
                rc |= emu_rv_conv(BM, 32, x.data(), C, B, T, F, C, w.data(), b.data(), k, N, 26, 1, 0, r.data(), N,
                                  o.data(), N);
                auto wu = vec((size_t)2 * 4 * C * 4 * 8), bu = vec(8), ou = vec((size_t)B * 2 * T * 2 * F * 8);
                rc |= emu_rv_conv(BM, 16, x.data(), C, B, T, F, C, wu.data(), bu.data(), 2, 32, 32, 1, 1, nullptr, 0,
                                  ou.data(), 8);
            }
    {
        const int B = 2, T = 5, F = 6;
        auto x = vec((size_t)B * T * F), sc = vec(1), sh = vec(1), w = vec(16 * 9), b = vec(16),
             o = vec((size_t)B * T * F * 16);
        rc |= emu_rv_conv_small(x.data(), T * F, F, 1, 1, B, T, F, 1, sc.data(), sh.data(), w.data(), b.data(), 3, 16,
                                1, 0, o.data(), 16);
        auto xh = vec((size_t)B * T * F * 16), wh = vec(3 * 16 * 9), bh = vec(3), oh = vec((size_t)B * T * 3 * F);
        rc |= emu_rv_conv_small(xh.data(), T * F * 16, F * 16, 16, 1, B, T, F, 16, nullptr, nullptr, wh.data(),
                                bh.data(), 3, 3, 0, 1, oh.data(), 0);
        auto xp = vec((size_t)B * T * F * 16), op = vec((size_t)B * (T / 2) * (F / 2) * 16);
        rc |= emu_rv_pool(xp.data(), 16, B, T, F, 16, op.data());
    }
    {                                                      // a full and a partial batch group
        const int B = 5, T = 1;
        auto xg = vec((size_t)B * T * 1536), whh = vec((size_t)2 * 768 * 256), bhh = vec(2 * 768),
             o = vec((size_t)B * T * 512);
        rc |= emu_rv_gru(xg.data(), whh.data(), bhh.data(), B, T, o.data());
    }
    {                                                      // 22050 -> 16000: 320 phases, a stride of 441 samples
        const int B = 2, N = 500, nw = 320, orig = 441, width = 179, taps = 2 * width + orig, n_out = (nw * N + orig - 1) / orig;
        auto x = vec((size_t)B * N), table = vec((size_t)nw * taps), o = vec((size_t)B * n_out);
        rc |= emu_rv_resample(x.data(), B, N, table.data(), nw, orig, taps, width, n_out, o.data());
    }
    for (int N : {513, 1101}) {
        const int B = 2, hop = 160, nf = 1 + N / hop, t_pad = 32;
        auto y = vec((size_t)B * N), win = vec(1024), basis = vec((size_t)128 * 513), o = vec((size_t)B * t_pad * 128);
        std::vector<int> lohi(256);
        for (int m = 0; m < 128; ++m) { lohi[2 * m] = 4 * m; lohi[2 * m + 1] = 4 * m + 5; }
        rc |= emu_rv_mel(y.data(), B, N, win.data(), basis.data(), lohi.data(), hop, nf, t_pad, o.data());
    }
    {
        auto sal = vec((size_t)2 * 9 * 360), f0 = vec((size_t)2 * 7);
        rc |= emu_rv_decode(sal.data(), 2, 9, 7, 0.03f, f0.data());
    }
    std::printf("done %d\n", rc);
    return rc;
}
#endif
