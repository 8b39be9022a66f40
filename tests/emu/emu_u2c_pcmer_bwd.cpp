// CPU execution of csrc/pcmer_bwd.cu's kernel sources (see host_emu.h).  Built by tests/test_emu_u2c_pcmer_backward.py.
// host_emu.h has no warp intrinsics, so __shfl_xor_sync is provided here: every thread of the emulated CTA writes its
// value to a slot, the CTA meets at a barrier, reads its partner's slot (lane ^ d stays inside the warp) and meets again.
// That needs every thread of the CTA to run the same sequence of shuffles, which the kernels guarantee (a warp past the
// last row clamps its row index and still joins them).
#define B2D_HOST_EMU 1
#include "host_emu.h"

namespace emu_shfl { inline float f[256]; inline int i[256]; }
inline float __shfl_xor_sync(unsigned, float v, int d) {
    emu_shfl::f[threadIdx.x] = v;
    emu::sync();
    const float r = emu_shfl::f[threadIdx.x ^ d];
    emu::sync();
    return r;
}
inline int __shfl_xor_sync(unsigned, int v, int d) {
    emu_shfl::i[threadIdx.x] = v;
    emu::sync();
    const int r = emu_shfl::i[threadIdx.x ^ d];
    emu::sync();
    return r;
}
inline float rsqrtf(float x) { return 1.0f / std::sqrt(x); }

#include "../../ddsp_svc_b200/csrc/pcmer_bwd.cu"

namespace { unsigned ctas(int rows) { return (unsigned)((rows + kRowsPerCta - 1) / kRowsPerCta); } }

extern "C" int emu_attn_readout_bwd(const float* g_out, const float* out, const float* d_inv, int B, int H, int T, float* gn) {
    const int rows = B * H * T;
    emu::launch(ctas(rows), 1u, 256, [&] { u2c_attn_readout_bwd_kernel(g_out, out, d_inv, H, T, rows, gn); });
    return 0;
}

extern "C" int emu_feat_bwd(float* g, const float* phi, const float* data, const float* vec, const float* scal, int rows, int T,
                            int J, int is_query, float eps, float* gx) {
    if (J > kJmax || rows % T) return -2;
    emu::launch(ctas(rows), 1u, 256, [&] { u2c_feat_bwd_kernel(g, phi, data, vec, is_query ? scal : nullptr, rows, T, J, is_query, eps, gx); });
    return 0;
}

extern "C" int emu_qkv_gather_bwd(const float* gq, const float* gk, const float* gv, const float* qkv, int B, int H, int T,
                                  int normalized, float* gqkv) {
    const int rows = B * H * T;
    emu::launch(ctas(rows), 1u, 256, [&] { u2c_qkv_gather_bwd_kernel(gq, gk, gv, qkv, H, T, rows, normalized, gqkv); });
    return 0;
}
