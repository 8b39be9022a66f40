// CPU execution of csrc/frontend.cu's kernel source (see host_emu.h).  Built by tests/test_emu_offline.py.  Each emu_*
// function fills the kernel's parameters as the matching b2d_* entry point does and launches the same grid.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#define gridDim (emu::grid_dim)
#define blockDim (emu::block_dim)

// the frontend kernels reduce fp64 across the warp: one double exchanged as its two 32-bit halves, two collectives
inline double __shfl_xor_sync(unsigned mask, double v, int d) {
    uint64_t u;
    std::memcpy(&u, &v, 8);
    const int lo = __shfl_xor_sync(mask, (int)(uint32_t)u, d), hi = __shfl_xor_sync(mask, (int)(uint32_t)(u >> 32), d);
    u = (uint64_t)(uint32_t)lo | ((uint64_t)(uint32_t)hi << 32);
    std::memcpy(&v, &u, 8);
    return v;
}

#include "../../ddsp_svc_b200/csrc/frontend.cu"

extern "C" int emu_slicer_rms(const float* audio, int64_t n_samples, int frame_length, int hop, float* rms) {
    const long long n_frames = 1 + ((long long)n_samples + 2 * (frame_length / 2) - frame_length) / hop;
    emu::launch((unsigned)((n_frames + 7) / 8), 1u, 256, [&] {
        slicer_rms_kernel(audio, n_samples, frame_length, hop, n_frames, rms);
    });
    return 0;
}

// grid: the entry point's (seg_len + 255) / 256 capped at 16 CTAs per SM; `grid` here lets a test force the grid-stride loop
extern "C" int emu_segment_place(float* result, const float* seg, int64_t seg_len, int64_t idx, int64_t fade_len,
                                 int grid) {
    emu::launch((unsigned)grid, 1u, 256, [&] { segment_place_kernel(result, seg, seg_len, idx, fade_len); });
    return 0;
}

extern "C" int emu_cross_fade(const float* a, int64_t len_a, const float* b, int64_t len_b, int64_t idx, float* out,
                              int grid) {
    emu::launch((unsigned)grid, 1u, 256, [&] { cross_fade_kernel(a, len_a, b, len_b, idx, out); });
    return 0;
}
