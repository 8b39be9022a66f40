// CPU execution of csrc/mel.cu's kernel sources (see host_emu.h).  Built by tests/test_emu_mel_backward.py.
// emu_mel_fwd runs mel_kernel, emu_mel_bwd runs mel_bwd_kernel with the caller's chunk length (the C entry point picks
// it from the SM count), so the tests can cut an utterance into many chunks or none.
#define B2D_HOST_EMU 1
#include "host_emu.h"
#include "../../ddsp_svc_b200/csrc/mel.cu"

namespace { alignas(16) unsigned char smem_raw[1 << 17]; }   // the kernels' `extern __shared__` array

namespace {
int pads(int T, int hop, int& pad_left, int& reflect) {
    pad_left = (kN - hop) / 2;
    int pad_right = (kN - hop + 1) / 2;
    if (kN - T - pad_left > pad_right) pad_right = kN - T - pad_left;
    reflect = pad_right < T ? 1 : 0;
    return b2d_mel_frames(T, kN, kN, hop);
}
}  // namespace

extern "C" int emu_mel_fwd(const float* y, const float* window, const float* basis, const int* lohi, int B, int T, int hop,
                           int n_mels, float clip, float* out) {
    static_assert(kSmemBytes <= sizeof(smem_raw), "shared-memory emulation buffer too small");
    MelParams p;
    p.y = y; p.window = window; p.basis = basis; p.lohi = lohi; p.out = out;
    p.T = T; p.hop = hop; p.n_mels = n_mels; p.clip = clip;
    p.n_frames = pads(T, hop, p.pad_left, p.reflect);
    if (p.n_frames <= 0) return -1;
    emu::launch((unsigned)((p.n_frames + kFramesPerCta - 1) / kFramesPerCta), (unsigned)B, kThreads, [&] { mel_kernel(p); });
    return 0;
}

extern "C" int emu_mel_bwd(const float* y, const float* window, const float* basis, const int* lohi, const int* bin_range,
                           const float* g, long long gs_b, long long gs_m, long long gs_f, int B, int T, int hop,
                           int n_mels, float clip, int chunk, float* dy) {
    static_assert(kBwdSmemFixed + kMaxChunk * sizeof(float) <= sizeof(smem_raw), "shared-memory emulation buffer too small");
    if (chunk <= 0 || chunk > kMaxChunk) return -2;
    MelBwdParams p;
    p.y = y; p.window = window; p.basis = basis; p.lohi = lohi; p.bin_range = bin_range;
    p.g = g; p.gs_b = gs_b; p.gs_m = gs_m; p.gs_f = gs_f; p.dy = dy;
    p.T = T; p.hop = hop; p.n_mels = n_mels; p.clip = clip; p.chunk = chunk;
    p.n_frames = pads(T, hop, p.pad_left, p.reflect);
    if (p.n_frames <= 0) return -1;
    emu::launch((unsigned)((T + chunk - 1) / chunk), (unsigned)B, kThreads, [&] { mel_bwd_kernel(p); });
    return 0;
}
