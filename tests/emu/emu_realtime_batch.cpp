// CPU execution of csrc/realtime.cu's batched entry points (see host_emu.h).  Built by tests/test_emu_realtime_batch.py,
// which compares every row with emu_realtime.cpp's single-session launch; with -DEMU_ASAN the main below runs them
// under AddressSanitizer, and tsan_realtime_batch.cpp includes it for ThreadSanitizer.  Each emu_* function fills the
// kernel's parameters as the matching b2d_rt_*_batch entry point does and launches the same grid.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#include "../../ddsp_svc_b200/csrc/realtime.cu"

namespace {
size_t align256(size_t bytes) { return (bytes + 255) / 256 * 256; }
}  // namespace

// b2d_rt_f0_regrid_workspace_bytes: one row's vsrc | vdst | prev
extern "C" size_t emu_rt_regrid_row_bytes(int n_src, int n_dst) {
    return align256((size_t)n_src * 8) + align256((size_t)n_dst * 8) + align256((size_t)std::max(n_src, n_dst) * 4);
}

extern "C" int emu_rt_f0_regrid_batch(const float* src, int rows, int n_src, double src_step, double src_div,
                                      float src_scale, int n_dst, int pad, double dst_step, int mode, double f0_min,
                                      const float* post_scale, float* out, void* workspace) {
    RtRegridParams p{};
    p.src = src; p.n_src = n_src; p.src_step = src_step; p.src_div = src_div; p.src_scale = src_scale;
    p.n_dst = n_dst; p.pad = pad; p.dst_step = dst_step; p.mode = mode; p.f0_min = f0_min; p.post_scale = 1.f;
    p.post_scale_rows = mode == 1 ? post_scale : nullptr;
    p.out = out;
    char* ws = static_cast<char*>(workspace);
    p.vsrc = reinterpret_cast<double*>(ws);
    p.vdst = reinterpret_cast<double*>(ws + align256((size_t)n_src * 8));
    p.prev = reinterpret_cast<int*>(ws + align256((size_t)n_src * 8) + align256((size_t)n_dst * 8));
    p.ws_stride = emu_rt_regrid_row_bytes(n_src, n_dst);
    emu::launch((unsigned)rows, 1u, kRegridThreads, [&] { rt_regrid_kernel(p); });
    return 0;
}

extern "C" int emu_rt_sola_batch(const float* x, long long x_stride, const float* buf, int rows, int crossfade,
                                 int search, int* shift) {
    emu::launch((unsigned)rows, 1u, kSolaThreads,
                [&] { rt_sola_batch_kernel(x, x_stride, buf, crossfade, search, shift); });
    return 0;
}

extern "C" int emu_rt_crossfade_batch(const float* x, long long x_stride, const int* shift, const float* buf, int rows,
                                      const float* fade_in, const float* fade_out, int block, int crossfade,
                                      int phase_vocoder, float* out, float* next_buf, float* bins) {
    RtCrossfadeParams p{x, shift, buf, fade_in, fade_out, block, crossfade, bins, out, next_buf, x_stride};
    const unsigned grid = (unsigned)((block + crossfade + kCrossfadeThreads - 1) / kCrossfadeThreads);
    if (phase_vocoder) {
        const int warps = kCrossfadeThreads / 32;
        emu::launch((unsigned)((crossfade / 2 + 1 + warps - 1) / warps), (unsigned)rows, kCrossfadeThreads,
                    [&] { rt_pv_bins_kernel(p); });
        emu::launch(grid, (unsigned)rows, kCrossfadeThreads, [&] { rt_crossfade_kernel<true>(p); });
    } else {
        emu::launch(grid, (unsigned)rows, kCrossfadeThreads, [&] { rt_crossfade_kernel<false>(p); });
    }
    return 0;
}

#ifdef EMU_ASAN
// Every input and output in a heap buffer of exactly its logical size: the last row of each ends at the end of its
// buffer, so a row offset or stride one too far is an AddressSanitizer report.  Values are arbitrary (the numerics are
// tests/test_emu_realtime_batch.py's business).
#include <memory>
#include <random>
#include <vector>
template <class T>
std::unique_ptr<T[]> heap(size_t n, std::mt19937& rng, float lo = -1.f, float hi = 1.f) {
    std::unique_ptr<T[]> p(new T[n]);
    std::uniform_real_distribution<float> ud(lo, hi);
    for (size_t i = 0; i < n; ++i) p[i] = (T)ud(rng);
    return p;
}
int main() {
    std::mt19937 rng(5);
    int rc = 0;
    for (int mode : {0, 1}) {
        const int rows = 3, n_src = 300, n_dst = 280;
        auto src = heap<float>((size_t)rows * n_src, rng, 0.f, 400.f);
        for (int i = 0; i < n_src; i += 3) src[(size_t)n_src + i] = 0.f;            // row 1 partly unvoiced
        auto post = heap<float>(rows, rng, 0.5f, 2.f);
        auto out = heap<float>((size_t)rows * n_dst, rng);
        std::unique_ptr<char[]> ws(new char[rows * emu_rt_regrid_row_bytes(n_src, n_dst)]);
        rc |= emu_rt_f0_regrid_batch(src.get(), rows, n_src, 0.01, mode ? 1.0 : 1.1, 1.1f, n_dst, mode ? 9 : 0,
                                     512.0 / 44100.0, mode, 50.0, post.get(), out.get(), ws.get());
    }
    const int rows = 4, cf = 200, search = 30, block = 150;
    {
        const long long stride = cf + search;
        auto x = heap<float>((size_t)rows * stride, rng);
        auto buf = heap<float>((size_t)rows * cf, rng);
        std::unique_ptr<int[]> shift(new int[rows]);
        rc |= emu_rt_sola_batch(x.get(), stride, buf.get(), rows, cf, search, shift.get());
    }
    for (int pv : {0, 1}) {
        const long long stride = search + block + cf;
        auto x = heap<float>((size_t)rows * stride, rng);
        auto buf = heap<float>((size_t)rows * cf, rng);
        auto fi = heap<float>(cf, rng, 0.f, 1.f), fo = heap<float>(cf, rng, 0.f, 1.f);
        std::unique_ptr<int[]> shift(new int[rows]);
        for (int r = 0; r < rows; ++r) shift[r] = r == rows - 1 ? search : r;
        auto out = heap<float>((size_t)rows * block, rng), nxt = heap<float>((size_t)rows * cf, rng);
        auto bins = heap<float>((size_t)rows * 3 * (cf / 2 + 1), rng);
        rc |= emu_rt_crossfade_batch(x.get(), stride, shift.get(), buf.get(), rows, fi.get(), fo.get(), block, cf, pv,
                                     out.get(), nxt.get(), bins.get());
    }
    std::printf("done %d\n", rc);
    return rc;
}
#endif
