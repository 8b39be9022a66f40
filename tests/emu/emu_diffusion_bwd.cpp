// CPU execution of csrc/diffusion_bwd.cu's kernel source (see host_emu.h).  Built by tests/test_emu_diffusion_backward.py.
// Every entry takes the launch's CTA and thread counts, so a test can run one kernel on different grids and compare
// the results bit for bit (the kernels stride over elements, slabs and columns by the grid and the block).
#define B2D_HOST_EMU 1
#include "host_emu.h"

namespace emu_dfb { inline dim3 grid_dim, block_dim; }
#define gridDim (emu_dfb::grid_dim)
#define blockDim (emu_dfb::block_dim)
inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }

#include "../../ddsp_svc_b200/csrc/diffusion_bwd.cu"

namespace {
void run(unsigned ctas, unsigned threads, const std::function<void()>& k) {
    emu_dfb::grid_dim.x = ctas;
    emu_dfb::block_dim.x = threads;
    emu::launch(ctas, 1, threads, k);
}
int slabs(int T) { return (T + kDfSlab - 1) / kDfSlab; }
}  // namespace

extern "C" {
int emu_df_slab(void) { return kDfSlab; }
void emu_df_loss_input(unsigned ctas, unsigned threads, const float* gt, const float* noise, const long long* t,
                       const float* sqrt_ac, const float* sqrt_1m_ac, int n_steps, float smin, float range, int B, int T,
                       int M, float* hi, float* lo) {
    run(ctas, threads, [&] {
        df_loss_input_kernel(gt, noise, t, sqrt_ac, sqrt_1m_ac, n_steps, smin, range, T, M, (size_t)B * T * M, hi, lo);
    });
}
void emu_df_relu_backward(unsigned ctas, unsigned threads, const float* gy, const float* pre, const float* bias, int n_rows,
                          int C, float* gx, float* hi, float* lo) {
    run(ctas, threads, [&] { df_relu_bwd_kernel(gy, pre, bias, C, (size_t)n_rows * C, gx, hi, lo); });
}
void emu_df_mish_backward(unsigned ctas, unsigned threads, const float* gy, const float* x, int n, float* gx, float* hi,
                          float* lo) {
    run(ctas, threads, [&] { df_mish_bwd_kernel(gy, x, (size_t)n, gx, hi, lo); });
}
void emu_df_gate_backward(unsigned ctas, unsigned threads, const float* ga, const float* g, const float* cond, int cond_stride,
                          int n_tokens, int C, int layer, int n_layers, float* gz, float* gz_hi, float* gz_lo) {
    run(ctas, threads, [&] {
        df_gate_bwd_kernel(ga, g, cond, cond_stride, C, 2 * C * n_layers, layer, (size_t)n_tokens * C, gz, gz_hi, gz_lo);
    });
}
// part: B slabs(T) C n_layers doubles (NULL with gu NULL)
void emu_df_layer_backward(unsigned ctas, unsigned threads, const float* gu, float* gh, const float* gsk, float skip_div,
                           int B, int T, int C, int layer, int n_layers, float* gr, float* gr_hi, float* gr_lo,
                           double* part) {
    run(ctas, threads, [&] {
        df_layer_bwd_kernel(gu, gh, gsk, skip_div, T, C, C * n_layers, layer, slabs(T), B * slabs(T), gr, gr_hi, gr_lo, part);
    });
}
}
