// CPU execution of csrc/hubert.cu's kernel source (see host_emu.h).  Built by tests/test_emu_hubert.py; the same test
// builds it with -DEMU_ASAN under AddressSanitizer (main below) and tsan_main.cpp includes it for ThreadSanitizer.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#define gridDim (emu::grid_dim)
#define blockDim (emu::block_dim)
#include "../../ddsp_svc_b200/csrc/hubert.cu"

namespace {
alignas(16) float4 smem4[(kPosSmem > kAttnSmem ? kPosSmem : kAttnSmem) / sizeof(float4)];   // `extern __shared__`
}  // namespace

extern "C" int emu_hb_conv0(const float* x, int B, int N, int pad, const float* w, int L0, int La, float* y,
                            double* part) {
    emu::launch((unsigned)((La + kConv0Tile - 1) / kConv0Tile), (unsigned)B, 256,
                [&] { hb_conv0_kernel(x, N, pad, w, L0, La, y, part); });
    return 0;
}

extern "C" int emu_hb_gn_finalize(const double* part, int B, int n_tiles, int L0, const float* gamma,
                                  const float* beta, float eps, float* scale, float* shift) {
    emu::launch((unsigned)((B * kC0 + 255) / 256), 1u, 256,
                [&] { hb_gn_finalize_kernel(part, B, n_tiles, L0, gamma, beta, eps, scale, shift); });
    return 0;
}

extern "C" int emu_hb_posconv(const float* x, int B, int T, const float* w, const float* bias, float* y) {
    emu::launch(dim3{(unsigned)((T + kPosBM - 1) / kPosBM), (unsigned)kPosGroups, (unsigned)B}, 256,
                [&] { hb_posconv_kernel(x, T, w, bias, y); });
    return 0;
}

extern "C" int emu_hb_attention(const float* qkv, int B, int T, float* hi, float* lo) {
    emu::launch(dim3{(unsigned)((T + kAttnQ - 1) / kAttnQ), (unsigned)kHeads, (unsigned)B}, 128,
                [&] { hb_attention_kernel(qkv, T, hi, lo); });
    return 0;
}

extern "C" int emu_hb_align(const float* units, int B, int T, int C, float ratio, int n_frames, float* out) {
    emu::launch(2u, 1u, 64u, [&] { hb_align_kernel(units, B, T, C, ratio, n_frames, out); });
    return 0;
}

extern "C" int emu_hb_act(const float* x, int rows, int C, int rows_per_b, const float* scale, const float* shift,
                          float* hi, float* lo) {
    emu::launch(3u, 1u, 64u, [&] { hb_act_kernel(x, (size_t)rows * C, C, rows_per_b, scale, shift, hi, lo); });
    return 0;
}

extern "C" int emu_hb_ln(const float* x, const float* y, int rows, int T, int rows_per_b, int C, int gelu,
                         const float* gamma, const float* beta, float eps, float* h, float* hi, float* lo) {
    const unsigned grid = (unsigned)((rows + 7) / 8);
    if (C == 512)
        emu::launch(grid, 1u, 256, [&] { hb_ln_kernel<16>(x, y, rows, T, rows_per_b, gelu, gamma, beta, eps, h, hi, lo); });
    else if (C == 768)
        emu::launch(grid, 1u, 256, [&] { hb_ln_kernel<24>(x, y, rows, T, rows_per_b, gelu, gamma, beta, eps, h, hi, lo); });
    else
        return -1;
    return 0;
}

#ifdef EMU_ASAN
// Every input in a heap buffer of exactly its logical size, at the edge shapes: any read or write past a tensor is an
// AddressSanitizer report.  Values are arbitrary (the numerics are tests/test_emu_hubert.py's business).
#include <random>
#include <vector>
int main() {
    std::mt19937 rng(7);
    std::uniform_real_distribution<float> ud(-1.f, 1.f);
    auto vec = [&](size_t n) { std::vector<float> v(n); for (auto& e : v) e = ud(rng); return v; };
    int rc = 0;
    for (int pad : {0, 40}) {
        const int B = 2, N = 400, L0 = (N + 2 * pad - 10) / 5 + 1, La = L0 + 2, tiles = (La + 63) / 64;
        auto x = vec((size_t)B * N), w = vec(512 * 10), y = vec((size_t)B * La * 512), g = vec(512), be = vec(512),
             sc = vec((size_t)B * 512), sh = vec((size_t)B * 512);
        std::vector<double> part((size_t)B * tiles * 2 * 512);
        rc |= emu_hb_conv0(x.data(), B, N, pad, w.data(), L0, La, y.data(), part.data());
        rc |= emu_hb_gn_finalize(part.data(), B, tiles, L0, g.data(), be.data(), 1e-5f, sc.data(), sh.data());
    }
    for (int T : {1, 65}) {
        auto qkv = vec((size_t)T * 3 * 768), hi = vec((size_t)T * 768), lo = vec((size_t)T * 768);
        rc |= emu_hb_attention(qkv.data(), 1, T, hi.data(), lo.data());
    }
    {
        const int T = 2;
        auto x = vec((size_t)T * 768), w = vec((size_t)16 * 128 * 48 * 48), b = vec(768), y = vec((size_t)T * 768);
        rc |= emu_hb_posconv(x.data(), 1, T, w.data(), b.data(), y.data());
        auto u = vec((size_t)2 * 5 * 8), o = vec((size_t)2 * 9 * 8);
        rc |= emu_hb_align(u.data(), 2, 5, 8, 0.5f, 9, o.data());
    }
    {
        const int B = 2, L = 5, C = 40;
        auto x = vec((size_t)B * L * C), sc = vec((size_t)B * C), sh = vec((size_t)B * C), hi = vec((size_t)B * L * C),
             lo = vec((size_t)B * L * C);
        rc |= emu_hb_act(x.data(), B * L, C, L, sc.data(), sh.data(), hi.data(), lo.data());
        rc |= emu_hb_act(x.data(), B * L, C, B * L, nullptr, nullptr, hi.data(), nullptr);
    }
    for (int C : {512, 768}) {                             // 11 rows, 8 per CTA: 5 warps of the second return
        const int B = 1, T = 11, per_b = C == 512 ? T + 3 : T;
        auto x = vec((size_t)B * per_b * C), y = vec((size_t)B * T * C), g = vec(C), b = vec(C),
             hi = vec((size_t)B * T * C), lo = vec((size_t)B * T * C);
        rc |= emu_hb_ln(x.data(), C == 768 ? y.data() : nullptr, B * T, T, per_b, C, C == 512, g.data(), b.data(),
                        1e-5f, C == 768 ? x.data() : nullptr, hi.data(), C == 768 ? lo.data() : nullptr);
    }
    std::printf("done %d\n", rc);
    return rc;
}
#endif
