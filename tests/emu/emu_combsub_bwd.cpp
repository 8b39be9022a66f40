// CPU execution of csrc/combsub_bwd.cu (the CombSub backward kernels, see host_emu.h).  Built by
// tests/test_emu_combsub_backward.py.  The caller passes the forward's comb, all-passed comb and harmonic impulse
// responses (the forward's kernels are not emulated here).
#define B2D_HOST_EMU 1
#include "host_emu.h"

inline void sincospi(double x, double* s, double* c) { *s = std::sin(M_PI * x); *c = std::cos(M_PI * x); }

#include "../../ddsp_svc_b200/csrc/combsub_bwd.cu"

namespace { alignas(16) unsigned char smem_raw[1 << 16]; }   // the kernels' `extern __shared__` array

extern "C" int emu_combsub_bwd(const float* f0, const float* c_gd, const float* c_hm, const float* c_nm,
                               long long stride, const float* comb, const float* allpassed, const float* ir_h,
                               const float* noise_in, unsigned long long seed, long long utt_off, const float* g,
                               const float* g_harm, const float* g_noise, int B, int nF, int Ma, int Mh, int Mn,
                               double sr, float* da, float* grad) {
    static_assert(sizeof(CsSmem) <= sizeof(smem_raw), "shared-memory emulation buffer too small");
    CsBwdParams p;
    p.comb = comb; p.allpassed = allpassed; p.noise_in = noise_in; p.seed = seed; p.utt_off = utt_off;
    p.ir_h = ir_h; p.f0 = f0; p.hw_num = 1.5f * (float)sr;
    p.c_gd = c_gd; p.c_hm = c_hm; p.c_nm = c_nm; p.ctrl_stride = stride;
    p.g = g; p.g_harm = g_harm; p.g_noise = g_noise;
    p.nF = nF; p.Ma = Ma; p.Mh = Mh; p.Mn = Mn; p.da = da; p.grad = grad;
    emu::launch((unsigned)nF, (unsigned)B, kThreads, [&] { combsub_bwd_kernel<1>(p); });
    emu::launch((unsigned)nF, (unsigned)B, kThreads, [&] { combsub_bwd_kernel<2>(p); });
    return 0;
}
