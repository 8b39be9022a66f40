// CPU execution of csrc/pcmer_bwd.cu's kernel sources (see host_emu.h).  Built by tests/test_emu_u2c_pcmer_backward.py.
#define B2D_HOST_EMU 1
#include "host_emu.h"

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
