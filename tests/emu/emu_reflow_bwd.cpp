// CPU execution of csrc/reflow_bwd.cu's kernel source (see host_emu.h).  Built by tests/test_emu_reflow_backward.py.
// Every entry takes the launch's CTA and thread counts, so a test can run one kernel on different grids and compare
// the results bit for bit (the kernels stride over elements, slabs and columns by the grid and the block).
#define B2D_HOST_EMU 1
#include "host_emu.h"

namespace emu_rf { inline dim3 grid_dim, block_dim; }
#define gridDim (emu_rf::grid_dim)
#define blockDim (emu_rf::block_dim)
using std::erff;

#include "../../ddsp_svc_b200/csrc/reflow_bwd.cu"

namespace {
void run(unsigned ctas, unsigned threads, const std::function<void()>& k) {
    emu_rf::grid_dim.x = ctas;
    emu_rf::block_dim.x = threads;
    emu::launch(ctas, 1, threads, k);
}
int slabs(int T) { return (T + kRfSlab - 1) / kRfSlab; }
}  // namespace

extern "C" {
int emu_rf_slab(void) { return kRfSlab; }
void emu_rf_loss_input(unsigned ctas, unsigned threads, const float* gt, const float* x0, const float* t, float smin, float range,
                       int B, int T, int M, float* target, float* hi, float* lo) {
    run(ctas, threads, [&] { rf_loss_input_kernel(gt, x0, t, smin, range, T, M, (size_t)B * T * M, target, hi, lo); });
}
// part: B slabs(T) M doubles, cols: M doubles
void emu_rf_loss(unsigned ctas, unsigned threads, const float* g, const float* bias, const float* target, const float* w, int B,
                 int T, int M, double* part, double* cols, float* loss) {
    const int n_items = B * slabs(T);
    run(ctas, threads, [&] { rf_loss_slabs_kernel(g, bias, target, w, T, M, slabs(T), n_items, part); });
    run(ctas, threads, [&] { rf_slab_reduce_kernel(part, 1, n_items, M, nullptr, cols); });
    run(1, 1, [&] { rf_loss_finish_kernel(cols, M, (double)B * T * M, loss); });
}
void emu_rf_loss_backward(unsigned ctas, unsigned threads, const float* g, const float* bias, const float* target, const float* w,
                          const float* g_loss, int B, int T, int M, float* gv, float* hi, float* lo) {
    const size_t n = (size_t)B * T * M;
    run(ctas, threads, [&] { rf_loss_bwd_kernel(g, bias, target, w, g_loss, 1.0 / (double)n, T, M, n, gv, hi, lo); });
}
void emu_rf_gelu_backward(unsigned ctas, unsigned threads, const float* gy, const float* pre, const float* bias, int n_rows,
                          int C, float* gx, float* hi, float* lo) {
    run(ctas, threads, [&] { rf_gelu_bwd_kernel(gy, pre, bias, C, (size_t)n_rows * C, gx, hi, lo); });
}
// part: B slabs(T) D n_layers doubles
void emu_rf_layer_backward(unsigned ctas, unsigned threads, const float* gz, float* gh, int B, int T, int D, int layer,
                           int n_layers, float* gh_hi, float* gh_lo, float* z, float* z_hi, float* z_lo, double* part) {
    run(ctas, threads, [&] {
        rf_layer_bwd_kernel(gz, gh, T, D, D * n_layers, layer, slabs(T), B * slabs(T), gh_hi, gh_lo, z, z_hi, z_lo, part);
    });
}
void emu_rf_step_sums(unsigned ctas, unsigned threads, const double* part, int B, int T, int cols, float* out) {
    run(ctas, threads, [&] { rf_slab_reduce_kernel(part, B, slabs(T), cols, out, nullptr); });
}
}
