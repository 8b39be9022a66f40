// Backward of the old CombSub synthesizer (api.cu b2d_combsub_synth) with respect to its three raw controls, for the
// training phase (infer=False): reference ddsp/vocoder.py:834-862, ddsp/core.py:120-182,240-270.  See DESIGN §4.5b.
//
// The forward chain is a = FIR(comb, h_ap), harmonic = FIR(a, h_h), noise = FIR(u, h_n), in the direct form of
// sins_bwd.cu (h_nF := h_{nF-1}).  With g_h = dL/dsignal + dL/dharmonic and g_n = dL/dsignal + dL/dnoise:
//   combsub_bwd_kernel, stage 1, one CTA per (frame f, utterance):
//       harmonic filter: dh_h = corr(g_h, allpassed); da = FIR^T(g_h, h_h) for hop f (the cascade's input gradient,
//       written to the backward workspace); un-roll dh_h, times this frame's dynamic window (the fp32 formula of
//       ir_build_tc.cu), adjoint of torch's c2r irfft, dc_h = Re(dH) exp(c_h);
//       noise filter: dh_n = corr(g_n, u) with u regenerated (or noise_in), Hann, irfft adjoint, dc_n = Re(dH) exp(c)/128;
//   combsub_bwd_kernel, stage 2 (needs da of hops f-1 .. f+1 and the tap overhang, so a second launch):
//       all-pass filter: dh_ap = corr(da, comb), irfft adjoint, dphi_j = Im(dH_j conj H_j), reverse cumsum,
//       * pi (1 - tanh^2 c).  No input gradient: the comb depends on f0 only, which is data.
// Up to 1024 taps (n_mag <= 513): a thread owns taps 4 t .. 4 t + 3 and 512 + 4 t .. 512 + 4 t + 3.
// Every gradient element and every da sample has exactly one owning thread, which sums its terms in a fixed order: no
// atomics, results independent of the grid, of b2d_set_overlap and of batch sharding (the noise is keyed by the global
// utterance index).
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "fir_adjoint.cuh"

namespace {

using b2d_firadj::kP;                        // block size the backward is built for
using b2d_firadj::kThreads;
constexpr int kMaxTaps = 1024;               // 2 (n_mag - 1), n_mag <= 513
constexpr int kMaxBins = kMaxTaps / 2 + 1;

struct CsBwdParams {
    const float* comb;        // [B, T] the forward's comb source
    const float* allpassed;   // [B, T] the forward's all-pass output
    const float* noise_in;    // [B, T] or nullptr: in-kernel Philox noise keyed by (seed, utt_off + b)
    unsigned long long seed;
    long long utt_off;
    const float* ir_h;        // [B, nF, Lh] the forward's harmonic impulse responses
    const float* f0;          // [B, nF] (dynamic window)
    float hw_num;             // 1.5 sr in fp32, as ir_build.cu
    const float* c_gd;        // raw controls, frame stride ctrl_stride
    const float* c_hm;
    const float* c_nm;
    long long ctrl_stride;
    const float* g;           // dL/dsignal, dL/dharmonic, dL/dnoise [B, T] (nullptr = zero)
    const float* g_harm;
    const float* g_noise;
    int nF, Ma, Mh, Mn;
    float* da;                // [B, T] dL/dallpassed (stage 1 writes it, stage 2 reads it)
    float* grad;              // dense [B, nF, Ma + Mh + Mn]
};

using CsSmem = b2d_firadj::FirSmem<kMaxTaps>;

// stage 1: harmonic filter (dh_h, da) and noise filter; stage 2: all-pass filter on da
template <int STAGE>
__global__ void __launch_bounds__(kThreads) combsub_bwd_kernel(CsBwdParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    CsSmem& s = *reinterpret_cast<CsSmem*>(smem_raw);
    const size_t frow = (size_t)blockIdx.y * p.nF + blockIdx.x;
    float* grow = p.grad + frow * (size_t)(p.Ma + p.Mh + p.Mn);
    b2d_firadj::FirArgs a{};
    a.nF = p.nF; a.seed = p.seed; a.utt_off = p.utt_off; a.grad_row = grow;
    if (STAGE == 1) {
        a.M = p.Mh; a.x = p.allpassed; a.g = p.g; a.g_add = p.g_harm; a.ir = p.ir_h; a.dx = p.da;
        a.f0 = p.f0 + frow; a.hw_num = p.hw_num;
        a.ctrl = p.c_hm + frow * (size_t)p.ctrl_stride; a.col = p.Ma;
        b2d_firadj::fir_adjoint<b2d_firadj::kHarmonic>(s, a);

        a.M = p.Mn; a.x = p.noise_in; a.g_add = p.g_noise; a.ir = nullptr; a.dx = nullptr;
        a.ctrl = p.c_nm + frow * (size_t)p.ctrl_stride; a.col = p.Ma + p.Mh;
        b2d_firadj::fir_adjoint<b2d_firadj::kNoise>(s, a);
    } else {
        a.M = p.Ma; a.x = p.comb; a.g = p.da;
        a.ctrl = p.c_gd + frow * (size_t)p.ctrl_stride; a.col = 0;
        b2d_firadj::fir_adjoint<b2d_firadj::kAllpass>(s, a);
    }
}

}  // namespace

#ifndef B2D_HOST_EMU
namespace {
template <int STAGE>
int stage_launch(const CsBwdParams& p, int B, cudaStream_t st) {
    auto kern = combsub_bwd_kernel<STAGE>;
    if (sizeof(CsSmem) > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CsSmem));
        if (e != cudaSuccess) return b2d::fail((int)e, "combsub_synth_backward: smem attr: %s", cudaGetErrorString(e));
    }
    kern<<<dim3((unsigned)p.nF, (unsigned)B), kThreads, sizeof(CsSmem), st>>>(p);
    return b2d::check_launch(STAGE == 1 ? "combsub_synth_backward: stage 1" : "combsub_synth_backward: stage 2");
}
}  // namespace

extern "C" size_t b2d_combsub_synth_backward_workspace_bytes(int B, int n_frames, int block) {
    if (B <= 0 || n_frames <= 0 || block <= 0) return 0;
    return b2d::align256((size_t)B * n_frames * block * 4);     // dL/dallpassed
}

extern "C" int b2d_combsub_synth_backward(const float* f0_frames, const float* c_group_delay, const float* c_harmonic,
                                          const float* c_noise, int64_t ctrl_stride, const float* noise_in,
                                          uint64_t seed, int64_t utterance_offset, const void* forward_workspace,
                                          const float* grad_signal, const float* grad_harmonic,
                                          const float* grad_noise, int B, int n_frames, int block, int n_mag_allpass,
                                          int n_mag_harmonic, int n_mag_noise, double sampling_rate, float* grad_ctrl,
                                          void* workspace, size_t workspace_bytes, void* stream) {
    if (!f0_frames || !c_group_delay || !c_harmonic || !c_noise || !forward_workspace || !grad_ctrl || !workspace)
        return b2d::fail(B2D_ERR_NULL, "combsub_synth_backward: null pointer");
    if (B <= 0 || n_frames <= 0 || block <= 0 || n_mag_allpass < 2 || n_mag_harmonic < 2 || n_mag_noise < 2 ||
        ctrl_stride < n_mag_allpass || ctrl_stride < n_mag_harmonic || ctrl_stride < n_mag_noise)
        return b2d::fail(B2D_ERR_SHAPE, "combsub_synth_backward: bad shape B=%d nF=%d block=%d Ma=%d Mh=%d Mn=%d "
                         "stride=%lld", B, n_frames, block, n_mag_allpass, n_mag_harmonic, n_mag_noise,
                         (long long)ctrl_stride);
    if (block != kP || n_mag_allpass > kMaxBins || n_mag_harmonic > kMaxBins || n_mag_noise > kMaxBins || B > 65535)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "combsub_synth_backward: built for block %d, n_mag <= %d, B <= 65535 "
                         "(got block %d, n_mag %d / %d / %d, B %d)", kP, kMaxBins, block, n_mag_allpass,
                         n_mag_harmonic, n_mag_noise, B);
    const size_t need = b2d_combsub_synth_backward_workspace_bytes(B, n_frames, block);
    if (workspace_bytes < need)
        return b2d::fail(B2D_ERR_WORKSPACE, "combsub_synth_backward: workspace %zu < %zu bytes", workspace_bytes, need);
    if ((reinterpret_cast<uintptr_t>(workspace) & 255u) || (reinterpret_cast<uintptr_t>(forward_workspace) & 255u) ||
        (noise_in && !b2d::aligned16(noise_in)) || (reinterpret_cast<uintptr_t>(grad_ctrl) & 3u))
        return b2d::fail(B2D_ERR_ALIGN, "combsub_synth_backward: workspaces must be 256-byte aligned, noise_in 16-byte "
                         "aligned");

    const b2d::CombSubWorkspace fw = b2d::combsub_workspace(B, n_frames, block, n_mag_allpass, n_mag_harmonic, n_mag_noise);
    CsBwdParams p;
    p.comb = b2d::ws_at(forward_workspace, fw.comb);
    p.allpassed = b2d::ws_at(forward_workspace, fw.allpassed);
    p.ir_h = b2d::ws_at(forward_workspace, fw.ir_h);
    p.noise_in = noise_in; p.seed = seed; p.utt_off = utterance_offset;
    p.f0 = f0_frames; p.hw_num = 1.5f * (float)sampling_rate;
    p.c_gd = c_group_delay; p.c_hm = c_harmonic; p.c_nm = c_noise; p.ctrl_stride = ctrl_stride;
    p.g = grad_signal; p.g_harm = grad_harmonic; p.g_noise = grad_noise;
    p.nF = n_frames; p.Ma = n_mag_allpass; p.Mh = n_mag_harmonic; p.Mn = n_mag_noise;
    p.da = static_cast<float*>(workspace); p.grad = grad_ctrl;
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = stage_launch<1>(p, B, st);
    if (rc) return rc;
    return stage_launch<2>(p, B, st);
}
#endif  // B2D_HOST_EMU
