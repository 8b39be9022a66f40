// ThreadSanitizer driver for the emulated kernels (built by tests/test_emu_tsan.py with -fsanitize=thread).
// A CUDA shared-memory race (missing / misplaced __syncthreads) is a data race between the std::threads of host_emu.h,
// which TSan reports; `racy` is the negative control proving that it does.
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#if defined(TSAN_FIRFFT)
#include "emu_ltv_fir_fft.cpp"
#elif defined(TSAN_CSFAST)
#include "emu_combsubfast.cpp"
#elif defined(TSAN_SUPERFAST)
#include "emu_superfast.cpp"
#elif defined(TSAN_LINATTN)
#include "emu_linear_attention.cpp"
#elif defined(TSAN_HIFIGAN)
#include "emu_hifigan.cpp"
#elif defined(TSAN_RMVPE_CONV) || defined(TSAN_RMVPE_GRU) || defined(TSAN_RMVPE_MEL)
#include "emu_rmvpe.cpp"
#elif defined(TSAN_HUBERT_ATTN) || defined(TSAN_HUBERT_POSCONV) || defined(TSAN_HUBERT_CONV0) || defined(TSAN_HUBERT_LN)
#include "emu_hubert.cpp"
#else
#define B2D_HOST_EMU 1
#include "host_emu.h"
namespace {
float shared_buf[128];
void racy_kernel(float* out, bool with_barrier) {
    const int tid = threadIdx.x;
    shared_buf[tid] = (float)tid;
    if (with_barrier) __syncthreads();
    out[tid] = shared_buf[(tid + 1) & 127];      // reads the neighbour's slot
}
}  // namespace
#endif

int main(int argc, char** argv) {
    std::mt19937 rng(1);
    std::normal_distribution<float> nd(0.f, 1.f);
    auto fill = [&](std::vector<float>& v, float scale, float shift = 0.f) { for (auto& e : v) e = nd(rng) * scale + shift; };
    double s = 0;
#if defined(TSAN_FIRFFT)
    const int B = 1, nF = 7, L = 510, T = nF * 512;
    std::vector<float> x1(B * T), x2(B * T), ir1(B * nF * L), ir2(B * nF * L), y1(B * T), y2(B * T), mix(B * T), add(B * T);
    fill(x1, 1.f); fill(x2, 1.f); fill(ir1, 0.05f); fill(ir2, 0.05f); fill(add, 1.f);
    emu_ltv_fir_fft(x1.data(), ir1.data(), L, y1.data(), x2.data(), ir2.data(), L, y2.data(), add.data(), mix.data(), 1, 0, B, nF, 4);
    emu_ltv_fir_fft(x1.data(), ir1.data(), L, y1.data(), nullptr, ir2.data(), 254, y2.data(), nullptr, mix.data(), 1, 0, B, nF, 32);
    emu_ltv_fir_fft(x1.data(), ir1.data(), L, y1.data(), nullptr, nullptr, 0, nullptr, nullptr, mix.data(), 1, 0, B, nF, 2);
    {   // 2048-point instance (1022 taps)
        std::vector<float> irl(B * nF * 1022);
        fill(irl, 0.03f);
        emu_ltv_fir_fft(x1.data(), irl.data(), 1022, y1.data(), nullptr, nullptr, 0, nullptr, nullptr, mix.data(), 1, 0, B, nF, 4);
    }
    for (float v : mix) s += v;
#elif defined(TSAN_CSFAST)
    const int B = 1, nF = 6, T = nF * 512, C = 3 * 513;
    std::vector<float> comb(B * T), noise(B * T), dense(B * nF * C), out(B * T);
    fill(comb, 1.f); fill(noise, 1.f); fill(dense, 0.3f, -1.f);
    emu_combsubfast(comb.data(), dense.data(), dense.data() + 513, dense.data() + 1026, C, noise.data(), 1, 0, B, nF, 4, out.data());
    emu_combsubfast(comb.data(), dense.data(), dense.data() + 513, dense.data() + 1026, C, nullptr, 1, 0, B, nF, 32, out.data());
    for (float v : out) s += v;
#elif defined(TSAN_LINATTN)
    const int B = 1, H = 2, T = 37, J = 266;
    std::vector<float> qf(B * H * T * J), kf(B * H * T * J), v(B * H * T * 64), out(B * T * H * 64);
    fill(qf, 0.1f, 0.5f); fill(kf, 0.1f, 0.5f); fill(v, 1.f);
    emu_linear_attention(qf.data(), kf.data(), v.data(), out.data(), B, H, T, J, 1e-8f);
    for (float e : out) s += e;
#elif defined(TSAN_SUPERFAST)
    const int B = 1, nF = 9, T = nF * 512, C = 4 * 1025;
    std::vector<float> par(B * nF * 4), noise(B * T), dense(B * nF * C), out(B * T);
    for (int k = 0; k < nF; ++k) { par[4 * k] = 0.005f + 0.0001f * k; par[4 * k + 1] = k + 1 < nF ? 0.0001f : 0.f; par[4 * k + 2] = 0.1f * k - (int)(0.1f * k); par[4 * k + 3] = 0.f; }
    fill(noise, 1.f); fill(dense, 0.3f, -1.f);
    emu_superfast(par.data(), dense.data(), dense.data() + 1025, dense.data() + 2050, dense.data() + 3075, C, noise.data(), 1, 0, B, nF, 5, out.data());
    emu_superfast(par.data(), dense.data(), dense.data() + 1025, dense.data() + 2050, dense.data() + 3075, C, nullptr, 1, 0, B, nF, 29, out.data());
    for (float v : out) s += v;
#elif defined(TSAN_HIFIGAN)
    // 3 chunks of C_in (both cp.async stages refilled), a 15-row halo, a T % BM tail; a transposed stage with its source
    const int B = 1, T = 70, C = 48, k = 11, d = 3, u = 2, Co = 16;
    std::vector<float> x(B * T * C), w(2 * k * C * C), b(C), r(B * T * C), o(B * T * C);
    std::vector<float> wt(2 * 3 * C * u * Co), src(B * T * u * 2), wn(Co * 4), bn(Co), ot(B * T * u * Co);
    fill(x, 1.f); fill(w, 0.05f); fill(b, 0.1f); fill(r, 1.f); fill(wt, 0.05f); fill(src, 1.f); fill(wn, 0.3f); fill(bn, 0.1f);
    emu_hg_conv(64, 16, x.data(), T * C, C, 1, B, T, C, w.data(), b.data(), k, d, C, 1, r.data(), r.data(), 2.f, 0,
                nullptr, nullptr, nullptr, 0, 0, 0, o.data());
    emu_hg_conv(64, 16, x.data(), T * C, C, 1, B, T, C, wt.data(), b.data(), 3, 1, u * Co, 1, nullptr, nullptr, 1.f, u,
                src.data(), wn.data(), bn.data(), 4, 2, 1, ot.data());
    for (float v : o) s += v;
    for (float v : ot) s += v;
#elif defined(TSAN_RMVPE_CONV)
    // 3 chunks of C_in, k 3 (a halo on both sides) at tF = F < BM / 4, T not a multiple of tT; the up convolution
    const int B = 1, T = 9, F = 4, C = 48, N = 32;
    std::vector<float> x(B * T * F * C), w(2 * 9 * C * N), b(N), o(B * T * F * N), wu(2 * 4 * C * N), ou(B * 4 * T * F * 8);
    fill(x, 1.f); fill(w, 0.05f); fill(b, 0.1f); fill(wu, 0.05f);
    emu_rv_conv(64, 32, x.data(), C, B, T, F, C, w.data(), b.data(), 3, N, 26, 1, 0, nullptr, 0, o.data(), N);
    emu_rv_conv(64, 16, x.data(), C, B, T, F, C, wu.data(), b.data(), 2, N, N, 0, 1, nullptr, 0, ou.data(), 8);
    for (float v : o) s += v;
    for (float v : ou) s += v;
#elif defined(TSAN_RMVPE_GRU)
    // one 8-CTA cluster per direction, a partial batch group, 3 steps through distributed shared memory
    const int B = 2, T = 3;
    std::vector<float> xg(B * T * 1536), whh(2 * 768 * 256), bhh(2 * 768), o(B * T * 512);
    fill(xg, 1.f); fill(whh, 0.05f); fill(bhh, 0.1f);
    emu_rv_gru(xg.data(), whh.data(), bhh.data(), B, T, o.data());
    for (float v : o) s += v;
#elif defined(TSAN_RMVPE_MEL)
    // the FFT's shared-memory passes, two frames per transform, an odd frame count and the zeroed padding frames
    const int B = 1, N = 1101, hop = 160, nf = 1 + N / hop, t_pad = 32;
    std::vector<float> y(B * N), win(1024), basis(128 * 513, 0.01f), o(B * t_pad * 128);
    std::vector<int> lohi(256);
    for (int m = 0; m < 128; ++m) { lohi[2 * m] = 4 * m; lohi[2 * m + 1] = 4 * m + 5; }
    fill(y, 0.3f); fill(win, 0.2f, 0.5f);
    emu_rv_mel(y.data(), B, N, win.data(), basis.data(), lohi.data(), hop, nf, t_pad, o.data());
    for (float v : o) s += v;
#elif defined(TSAN_HUBERT_LN)
    // in place (h == x) with y, 11 rows at 8 per CTA: 5 warps of the second CTA return before any shuffle
    const int B = 1, T = 11, C = 768;
    std::vector<float> x(B * T * C), y(B * T * C), g(C), b(C), hi(B * T * C), lo(B * T * C);
    fill(x, 1.f); fill(y, 1.f); fill(g, 0.1f, 1.f); fill(b, 0.1f);
    emu_hb_ln(x.data(), y.data(), B * T, T, T, C, 0, g.data(), b.data(), 1e-5f, x.data(), hi.data(), lo.data());
    for (float v : x) s += v;
#elif defined(TSAN_HUBERT_ATTN)
    const int B = 1, T = 70;                                 // two key tiles, the second masked past T
    std::vector<float> qkv(B * T * 3 * 768), hi(B * T * 768), lo(B * T * 768);
    fill(qkv, 1.f);
    emu_hb_attention(qkv.data(), B, T, hi.data(), lo.data());
    for (float v : hi) s += v;
#elif defined(TSAN_HUBERT_POSCONV)
    const int B = 1, T = 3;
    std::vector<float> x(B * T * 768), w(16 * 128 * 48 * 48), b(768), y(B * T * 768);
    fill(x, 1.f); fill(w, 0.01f); fill(b, 0.1f);
    emu_hb_posconv(x.data(), B, T, w.data(), b.data(), y.data());
    for (float v : y) s += v;
#elif defined(TSAN_HUBERT_CONV0)
    const int B = 1, N = 1600, pad = 40, L0 = (N + 2 * pad - 10) / 5 + 1, La = L0 + 3;
    const int tiles = (La + 63) / 64;
    std::vector<float> x(B * N), w(512 * 10), y(B * La * 512);
    std::vector<double> part(B * tiles * 2 * 512);
    fill(x, 1.f); fill(w, 0.1f);
    emu_hb_conv0(x.data(), B, N, pad, w.data(), L0, La, y.data(), part.data());
    for (float v : y) s += v;
#else
    const bool with_barrier = argc > 1 && std::string(argv[1]) == "ok";
    std::vector<float> out(128);
    emu::launch(1, 1, 128, [&] { racy_kernel(out.data(), with_barrier); });
    for (float v : out) s += v;
#endif
    std::printf("done %g\n", s);
    return 0;
}
