// CPU execution of csrc/sins_bwd.cu (the Sins backward kernels, see host_emu.h).  Built by
// tests/test_emu_sins_backward.py.  The caller passes the forward's sinusoids and impulse responses (the bank and the
// impulse-response kernels use TMA / wgmma and are not emulated) and the fp64 frame phase of the phase scan.
#define B2D_HOST_EMU 1
#include "host_emu.h"

inline void sincospi(double x, double* s, double* c) { *s = std::sin(M_PI * x); *c = std::cos(M_PI * x); }

#include "../../ddsp_svc_b200/csrc/sins_bwd.cu"

namespace { alignas(16) unsigned char smem_raw[1 << 16]; }   // the kernels' `extern __shared__` array

extern "C" int emu_sins_bwd(const float* f0, const double* frame_phase, const float* c_amp, const float* c_gd,
                            const float* c_nm, long long stride, const float* sinus, const float* ir_ap,
                            const float* ir_n, const float* noise_in, unsigned long long seed, long long utt_off,
                            const float* g, const float* g_harm, const float* g_noise, int B, int nF, int H, int Ma,
                            int Mn, double sr, float* dx, float* grad) {
    static_assert(sizeof(FirSmem) <= sizeof(smem_raw) && sizeof(BankSmem) <= sizeof(smem_raw),
                  "shared-memory emulation buffer too small");
    FirBwdParams fp;
    fp.sinus = sinus; fp.noise_in = noise_in; fp.seed = seed; fp.utt_off = utt_off;
    fp.ir_ap = ir_ap; fp.ir_n = ir_n; fp.c_gd = c_gd; fp.c_nm = c_nm; fp.ctrl_stride = stride;
    fp.g = g; fp.g_harm = g_harm; fp.g_noise = g_noise;
    fp.nF = nF; fp.Ma = Ma; fp.Mn = Mn; fp.H = H; fp.dx = dx; fp.grad = grad;
    emu::launch((unsigned)nF, (unsigned)B, kThreads, [&] { sins_fir_bwd_kernel(fp); });

    BankBwdParams bp;
    bp.f0 = f0; bp.frame_phase = frame_phase; bp.c_amp = c_amp; bp.ctrl_stride = stride; bp.dx = dx;
    bp.nF = nF; bp.H = H; bp.inv_sr = 1.0 / sr; bp.nyquist = (float)(sr / 2.0);
    bp.grad = grad; bp.grad_stride = (long long)H + Ma + Mn;
    const auto run = [&](auto kern) { emu::launch((unsigned)nF, (unsigned)B, kThreads, [&] { kern(bp); }); };
    switch ((H + 127) / 128) {
        case 1: run(sins_bank_bwd_kernel<1>); break;
        case 2: run(sins_bank_bwd_kernel<2>); break;
        case 3: run(sins_bank_bwd_kernel<3>); break;
        default: run(sins_bank_bwd_kernel<4>); break;
    }
    return 0;
}
