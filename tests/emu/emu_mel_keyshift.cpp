// CPU execution of csrc/mel.cu's keyshift kernel source (see host_emu.h).  Built by tests/test_keyshift_mel.py.
// emu_mel_keyshift sets the shape up with the library's own keyshift_setup and launches mel_keyshift_kernel with the
// transform size and zero-upper choice of b2d_mel_spectrogram_keyshift.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#include "../../ddsp_svc_b200/csrc/mel.cu"

namespace { alignas(16) unsigned char smem_raw[1 << 17]; }   // the kernels' `extern __shared__` array

namespace {
template <int M, bool ZU> void run(const MelKeyshiftParams& p, int B) {
    static_assert(keyshift_smem_bytes<M>() <= sizeof(smem_raw), "shared-memory emulation buffer too small");
    emu::launch((unsigned)((p.n_frames + 1) / 2), (unsigned)B, kThreads, [&] { mel_keyshift_kernel<M, ZU>(p); });
}
}  // namespace

extern "C" int emu_mel_keyshift(const float* y, const float* table, const float* basis, const int* lohi, int B, int T,
                                int n_fft, int hop, int n_mels, float clip, float* out) {
    if (n_fft < hop || n_fft > kKeyshiftMaxN) return -4;
    MelKeyshiftParams p;
    p.y = y; p.table = table; p.basis = basis; p.lohi = lohi; p.out = out; p.n_mels = n_mels; p.clip = clip;
    if (keyshift_setup(p, T, n_fft, hop) <= 0) return -2;
    const int M = bluestein_size(n_fft, p.K);
    const bool zu = 2 * n_fft <= M;
    if (M == 1024) zu ? run<1024, true>(p, B) : run<1024, false>(p, B);
    else if (M == 2048) zu ? run<2048, true>(p, B) : run<2048, false>(p, B);
    else zu ? run<4096, true>(p, B) : run<4096, false>(p, B);
    return 0;
}

extern "C" int emu_mel_keyshift_frames(int T, int n_fft, int hop) {
    MelKeyshiftParams p;
    return keyshift_setup(p, T, n_fft, hop);
}
