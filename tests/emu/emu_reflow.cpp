// CPU execution of csrc/reflow.cu's kernel source (see host_emu.h).  Built by tests/test_emu_reflow.py.  The kernels
// are grid-stride loops: each entry runs them on a small fixed grid (3 CTAs of 32 threads) so every thread takes several
// elements and the loop bounds are exercised.
#define B2D_HOST_EMU 1
#include "host_emu.h"

namespace emu_rf { inline dim3 grid_dim, block_dim; }
#define gridDim (emu_rf::grid_dim)
#define blockDim (emu_rf::block_dim)
using std::erff;

#include "../../ddsp_svc_b200/csrc/reflow.cu"

namespace {
constexpr unsigned kCtas = 3, kThreads = 32;
void run(const std::function<void()>& k) {
    emu_rf::grid_dim.x = kCtas;
    emu_rf::block_dim.x = kThreads;
    emu::launch(kCtas, 1, kThreads, k);
}
}  // namespace

extern "C" {
int emu_rf_start(const float* noise, const float* gt, float ts, float one_m_ts, float smin, float range, int B, int T, int M,
                 float* x, float* hi, float* lo) {
    run([&] { rf_start_kernel(noise, gt, ts, one_m_ts, smin, range, T, M, (size_t)B * T * M, x, hi, lo); });
    return 0;
}
int emu_rf_layer_input(const float* g, const float* bias, float* h, int residual, const float* step, int step_stride,
                       const float* cond, int cond_stride, int B, int T, int D, float* hi, float* lo) {
    if (D % 4) return -3;
    run([&] {
        rf_layer_input_kernel(reinterpret_cast<const float4*>(g), reinterpret_cast<const float4*>(bias),
                              reinterpret_cast<float4*>(h), residual, step, step_stride, cond, cond_stride, T, D / 4,
                              (size_t)B * T * (D / 4), hi, lo);
    });
    return 0;
}
int emu_rf_ode(const float* g, const float* bias, float* x, float* acc, int stage, float dt, int n_tokens, int M, float* hi,
               float* lo) {
    run([&] { rf_ode_kernel(g, bias, x, acc, stage, dt, M, (size_t)n_tokens * M, hi, lo); });
    return 0;
}
int emu_rf_finish(const float* x, float smin, float range, int n, float* out) {
    run([&] { rf_finish_kernel(x, smin, range, (size_t)n, out); });
    return 0;
}
}
