// CPU execution of csrc/rss_loss.cu's kernel sources (see host_emu.h).  Built by tests/test_emu_rss_loss.py.
// emu_rss_forward runs rss_fwd_kernel for every scale and then rss_finalize_kernel; emu_rss_backward runs
// rss_bwd_kernel for every scale in order (the first stores, the others add), as the C entry points launch them.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#include "../../ddsp_svc_b200/csrc/rss_loss.cu"

namespace { alignas(16) unsigned char smem_raw[1 << 17]; }   // the kernels' `extern __shared__` array

namespace {
template <class F> void by_size(int n, F f) {
    const int M = bluestein_size(n);
    if (M == 1024) f(std::integral_constant<int, 1024>());
    else if (M == 2048) f(std::integral_constant<int, 2048>());
    else f(std::integral_constant<int, 4096>());
}
}  // namespace

extern "C" long long emu_rss_workspace_doubles(int B, int T, int n_scale, const int* n_ffts) {
    long long d = 0;
    for (int s = 0; s < n_scale; ++s) d += (long long)B * b2d_rss_frames(T, n_ffts[s]) * 3;
    return d;
}

extern "C" int emu_rss_forward(const float* xp, const float* xt, int B, int T, int n_scale, const int* n_ffts,
                               const float* const* tables, float alpha, float eps, double* part, double* norms,
                               float* loss) {
    static_assert(smem_bytes<4096>() <= sizeof(smem_raw), "shared-memory emulation buffer too small");
    if (n_scale <= 0 || n_scale > kMaxScales) return -2;
    RssFinalizeParams fp;
    fp.part = part; fp.norms = norms; fp.loss = loss; fp.B = B; fp.n_scale = n_scale; fp.alpha = alpha;
    long long off = 0;
    for (int s = 0; s < n_scale; ++s) {
        RssParams p = {};
        p.xp = xp; p.xt = xt; p.table = tables[s]; p.part = part + off;
        p.T = T; p.n = n_ffts[s]; p.F = b2d_rss_frames(T, p.n); p.B = B; p.alpha = alpha; p.eps = eps;
        if (p.F <= 0) return -2;
        fp.off[s] = off; fp.F[s] = p.F; fp.K[s] = p.n / 2 + 1;
        off += (long long)B * p.F * 3;
        by_size(p.n, [&](auto m) {
            constexpr int M = decltype(m)::value;
            emu::launch((unsigned)p.F, (unsigned)B, kThreads, [&] { rss_fwd_kernel<M>(p); });
        });
    }
    emu::launch(1, 1, kThreads, [&] { rss_finalize_kernel(fp); });
    return 0;
}

extern "C" int emu_rss_backward(const float* xp, const float* xt, int B, int T, int n_scale, const int* n_ffts,
                                const float* const* tables, float alpha, float eps, const double* norms,
                                const float* grad_loss, float* dx) {
    for (int s = 0; s < n_scale; ++s) {
        RssParams p = {};
        p.xp = xp; p.xt = xt; p.table = tables[s]; p.norms = norms + (size_t)s * B * 2; p.grad_loss = grad_loss;
        p.dx = dx; p.T = T; p.n = n_ffts[s]; p.F = b2d_rss_frames(T, p.n); p.B = B; p.accumulate = s > 0;
        p.alpha = alpha; p.eps = eps; p.inv_scales = 1.0 / n_scale;
        if (p.F <= 0) return -2;
        by_size(p.n, [&](auto m) {
            constexpr int M = decltype(m)::value;
            emu::launch((unsigned)p.F, (unsigned)B, kThreads, [&] { rss_bwd_kernel<M>(p); });
        });
    }
    return 0;
}

// S_p and S_t of every bin of every frame as the kernels compute them (the forward's transform_frames, bluestein_out and
// spec_bin), [B, F, K] each: lets the tests count the bins where the kernels' sign(log S_t - log S_p) differs from
// float64.
namespace {
template <int M> void spectra_kernel(const RssParams& p, float* sp, float* st) {
    const Smem<M> sm(smem_raw);
    const int tid = threadIdx.x, b = blockIdx.y, f = blockIdx.x, K = p.n / 2 + 1;
    const float2* chirp = reinterpret_cast<const float2*>(p.table + chirp_off(p.n));
    const float c = p.table[0];
    transform_frames<M>(sm, p, b, f, tid);
    for (int k = tid; k < K; k += kThreads) {
        const size_t o = ((size_t)b * p.F + f) * K + k;
        sp[o] = spec_bin(bluestein_out<M>(sm.z0, chirp, k), c, p.eps).S;
        st[o] = spec_bin(bluestein_out<M>(sm.z1, chirp, k), c, p.eps).S;
    }
}
}  // namespace

extern "C" int emu_rss_spectra(const float* xp, const float* xt, int B, int T, int n, const float* table, float eps,
                               float* sp, float* st) {
    RssParams p = {};
    p.xp = xp; p.xt = xt; p.table = table; p.T = T; p.n = n; p.F = b2d_rss_frames(T, n); p.B = B; p.eps = eps;
    if (p.F <= 0) return -2;
    by_size(n, [&](auto m) {
        constexpr int M = decltype(m)::value;
        emu::launch((unsigned)p.F, (unsigned)B, kThreads, [&] { spectra_kernel<M>(p, sp, st); });
    });
    return 0;
}
