// CPU execution of csrc/realtime.cu's kernel source (see host_emu.h).  Built by tests/test_realtime.py.  Each emu_*
// function fills the kernel's parameters as the matching b2d_rt_* entry point does and launches the same grid.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#include "../../ddsp_svc_b200/csrc/realtime.cu"

extern "C" int emu_rt_f0_regrid(const float* src, int n_src, double src_step, double src_div, float src_scale,
                                int n_dst, int pad, double dst_step, int mode, double f0_min, float post_scale,
                                float* out, double* vsrc, double* vdst, int* prev) {
    RtRegridParams p{};
    p.src = src; p.n_src = n_src; p.src_step = src_step; p.src_div = src_div; p.src_scale = src_scale;
    p.n_dst = n_dst; p.pad = pad; p.dst_step = dst_step; p.mode = mode; p.f0_min = f0_min; p.post_scale = post_scale;
    p.out = out; p.vsrc = vsrc; p.vdst = vdst; p.prev = prev;
    emu::launch(1u, 1u, kRegridThreads, [&] { rt_regrid_kernel(p); });
    return 0;
}

extern "C" int emu_rt_sola(const float* x, const float* buf, int crossfade, int search, int* shift) {
    emu::launch(1u, 1u, kSolaThreads, [&] { rt_sola_kernel(x, buf, crossfade, search, shift); });
    return 0;
}

extern "C" int emu_rt_crossfade(const float* x, const int* shift, const float* buf, const float* fade_in,
                                const float* fade_out, int block, int crossfade, int phase_vocoder, float* out,
                                float* next_buf, float* bins) {
    RtCrossfadeParams p{x, shift, buf, fade_in, fade_out, block, crossfade, bins, out, next_buf};
    const unsigned grid = (unsigned)((block + crossfade + kCrossfadeThreads - 1) / kCrossfadeThreads);
    if (phase_vocoder) {
        const int warps = kCrossfadeThreads / 32;
        emu::launch((unsigned)((crossfade / 2 + 1 + warps - 1) / warps), 1u, kCrossfadeThreads,
                    [&] { rt_pv_bins_kernel(p); });
        emu::launch(grid, 1u, kCrossfadeThreads, [&] { rt_crossfade_kernel<true>(p); });
    } else {
        emu::launch(grid, 1u, kCrossfadeThreads, [&] { rt_crossfade_kernel<false>(p); });
    }
    return 0;
}
