// CPU execution of csrc/superfast.cu's backward kernel source (see host_emu.h).  Built by
// tests/test_emu_superfast_backward.py.  The caller passes frame_par = (s, ds, acc_prev, 0) per frame (the frame scan
// uses warp shuffles and is not emulated).
#define B2D_HOST_EMU 1
#include "host_emu.h"
#include "../../ddsp_svc_b200/csrc/superfast.cu"

namespace { alignas(16) unsigned char smem_raw[1 << 17]; }   // the kernel's `extern __shared__` array

extern "C" int emu_superfast_bwd(const float* frame_par, const float* hm, const float* hp, const float* nm,
                                 const float* np_, long long stride, const float* noise_in, unsigned long long seed,
                                 long long utt_off, const float* grad, int B, int nF, int G, float* grad_ctrl) {
    static_assert(kSmemBytes <= sizeof(smem_raw), "shared-memory emulation buffer too small");
    SfBwdParams p;
    p.frame_par = reinterpret_cast<const float4*>(frame_par);
    p.c_hm = hm; p.c_hp = hp; p.c_nm = nm; p.c_np = np_; p.ctrl_stride = stride; p.noise_in = noise_in;
    p.grad = grad; p.grad_ctrl = grad_ctrl;
    p.nF = nF; p.P = 512; p.G = G; p.seed = seed; p.utt_off = utt_off;
    emu::launch((unsigned)((nF + G - 1) / G), (unsigned)B, kThreads, [&] { superfast_bwd_kernel<false>(p); });
    return 0;
}
