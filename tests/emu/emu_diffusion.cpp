// CPU execution of csrc/diffusion.cu's kernel source (see host_emu.h).  Built by tests/test_emu_diffusion.py.  The
// kernels are grid-stride loops: each entry runs them on a small fixed grid (3 CTAs of 32 threads) so every thread takes
// several elements and the loop bounds are exercised.
#define B2D_HOST_EMU 1
#include "host_emu.h"

namespace emu_df { inline dim3 grid_dim, block_dim; }
#define gridDim (emu_df::grid_dim)
#define blockDim (emu_df::block_dim)

#include "../../ddsp_svc_b200/csrc/diffusion.cu"

namespace {
constexpr unsigned kCtas = 3, kThreads = 32;
void run(const std::function<void()>& k) {
    emu_df::grid_dim.x = kCtas;
    emu_df::block_dim.x = kThreads;
    emu::launch(kCtas, 1, kThreads, k);
}
}  // namespace

extern "C" {
int emu_df_layer(const float* g, const float* bias, float* h, float* skip, int stage, const float* step, int step_stride,
                 float skip_div, int B, int T, int C, float* hi, float* lo) {
    if (C % 4) return -3;
    run([&] {
        df_layer_kernel(reinterpret_cast<const float4*>(g), reinterpret_cast<const float4*>(bias), reinterpret_cast<float4*>(h),
                        reinterpret_cast<float4*>(skip), stage, step, step_stride, skip_div, T, C / 4, (size_t)B * T * (C / 4),
                        hi, lo);
    });
    return 0;
}
int emu_df_gate(const float* g, const float* cond, int cond_stride, int n_tokens, int C, float* hi, float* lo) {
    if (C % 4) return -3;
    run([&] { df_gate_kernel(reinterpret_cast<const float4*>(g), cond, cond_stride, C / 4, (size_t)n_tokens * (C / 4), hi, lo); });
    return 0;
}
int emu_df_relu(const float* g, const float* bias, int n_tokens, int C, float* hi, float* lo) {
    if (C % 4) return -3;
    run([&] {
        df_relu_kernel(reinterpret_cast<const float4*>(g), reinterpret_cast<const float4*>(bias), C / 4,
                       (size_t)n_tokens * (C / 4), hi, lo);
    });
    return 0;
}
int emu_df_update(const float* g, const float* bias, const float* coef, const float* x, float* d_out, const float* h1,
                  const float* h2, const float* h3, const float* noise, int B, int T, int M, float* x_out, float* hi,
                  float* lo) {
    run([&] { df_update_kernel(g, bias, coef, x, d_out, h1, h2, h3, noise, T, M, (size_t)B * T * M, x_out, hi, lo); });
    return 0;
}
}
