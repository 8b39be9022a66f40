// CPU execution of csrc/combsubfast.cu's backward kernel source (see host_emu.h).  Built by
// tests/test_emu_combsubfast_backward.py.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#include "../../ddsp_svc_b200/csrc/combsubfast.cu"

namespace { alignas(16) unsigned char smem_raw[1 << 17]; }   // the kernel's `extern __shared__` array

extern "C" int emu_combsubfast_bwd(const float* comb, const float* hm, const float* hp, const float* nm, long long stride,
                                   const float* noise_in, unsigned long long seed, long long utt_off, const float* grad,
                                   int B, int nF, int G, float* grad_ctrl) {
    static_assert(kBwdSmemBytes <= sizeof(smem_raw), "shared-memory emulation buffer too small");
    CfBwdParams p;
    p.comb = comb; p.noise_in = noise_in; p.c_hm = hm; p.c_hp = hp; p.c_nm = nm; p.ctrl_stride = stride;
    p.grad = grad; p.grad_ctrl = grad_ctrl; p.nF = nF; p.G = G; p.seed = seed; p.utt_off = utt_off;
    emu::launch((unsigned)((nF + G - 1) / G), (unsigned)B, kThreads, [&] { combsubfast_bwd_kernel<false>(p); });
    return 0;
}
