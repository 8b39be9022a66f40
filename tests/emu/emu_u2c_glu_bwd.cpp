// CPU execution of csrc/unit2control_bwd.cu's GLU -> depthwise conv -> SiLU backward kernel source (see host_emu.h).
// Built by tests/test_emu_u2c_backward.py.  The second stage (the slabs added in order in fp64) is restated here: on
// the device it is u2c_reduce_partials_kernel.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#include "../../ddsp_svc_b200/csrc/unit2control_bwd.cu"

namespace { alignas(16) unsigned char smem_raw[1 << 17]; }   // the kernel's `extern __shared__` array

extern "C" int emu_u2c_glu_bwd(const float* h, const float* w, const float* bias, const float* gout, float* gh, float* dwb,
                               int B, int T, int Ci) {
    static_assert(kGluSmemBytes <= (int)sizeof(smem_raw), "shared-memory emulation buffer too small");
    if (B <= 0 || T <= 0 || Ci <= 0 || Ci % 128) return -2;
    const int n_tiles = (T + kDwTile - 1) / kDwTile;
    std::vector<float> part((size_t)B * n_tiles * Ci * kDwbStride, NAN);
    emu::launch((unsigned)(n_tiles * (Ci / 128)), (unsigned)B, 128,
                [&] { u2c_glu_bwd_kernel(h, w, bias, gout, gh, part.data(), T, Ci, n_tiles); });
    const size_t n = (size_t)Ci * kDwbStride;
    for (size_t j = 0; j < n; ++j) {
        double s = 0.0;
        for (int i = 0; i < B * n_tiles; ++i) s += (double)part[(size_t)i * n + j];
        dwb[j] = (float)s;
    }
    return 0;
}
