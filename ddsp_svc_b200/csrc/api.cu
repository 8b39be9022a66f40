// C-ABI plumbing of libb200ddsp: version, thread-local error string, and the drivers that
// chain the kernels of one synthesizer on the caller's stream.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "b2d_common.cuh"

namespace b2d {

char* err_buf() {
    static thread_local char buf[512] = {0};
    return buf;
}

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(err_buf(), 512, fmt, ap);
    va_end(ap);
    return code;
}

int ltv_fir_launch(const float* x1, const float* ir1, int taps1, float* y1, const float* x2, const float* ir2,
                   int taps2, float* y2, const float* addend, float* mix, uint64_t seed, int64_t utt_off, int B,
                   int nF, int P, cudaStream_t st);

bool fir_fft_selected();
bool fir_spec_supported(int P, int taps1, int taps2);
int ir_spectrum_launch(const float* ir1, int taps1, float* spec1, const float* ir2, int taps2, float* spec2, int B, int nF,
                       cudaStream_t st);
int ltv_fir_fft_spec_launch(const float* x1, const float* spec1, int taps1, float* y1, const float* x2, const float* spec2,
                            int taps2, float* y2, float* mix, uint64_t seed, int64_t utt_off, int B, int nF, int P, cudaStream_t st);
bool sins_fused_supported(int P, int taps_allpass, int taps_noise, int H);
int sins_fused_launch(const float* f0, const double* frame_phase, const float* c_amp, int64_t ctrl_stride, int H,
                      double sampling_rate, int round_fp32, const float* ir_allpass, int taps_allpass, float* harmonic,
                      const float* noise_in, const float* ir_noise, int taps_noise, float* noise_out, float* signal,
                      uint64_t seed, int64_t utt_off, int B, int nF, int P, cudaStream_t st);

int num_sms() {
    static std::atomic<int> cache[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { cudaGetLastError(); return 132; }
    int n = cache[dev].load(std::memory_order_relaxed);
    if (n <= 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { cudaGetLastError(); n = 132; }
        cache[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}

}  // namespace b2d

namespace b2d {
// The "packed" instantiations are the default (on Hopper they compile to the same scalar additions as the others).
// B2D_FFT_ARITH=scalar in the environment picks the scalar instantiations as the initial value
// (whole-suite A/B runs); b2d_set_fft_arith overrides at run time.
static int fft_arith_default() {
    const char* e = getenv("B2D_FFT_ARITH");
    return (e && !strcmp(e, "scalar")) ? 0 : 1;
}
std::atomic<int> g_fft_packed{fft_arith_default()};
}

// ---------------------------------------------------------------------------------------
// Fork/join inside one synthesizer call.  The impulse-response builds depend only on the raw controls, the oscillator
// bank / comb source only on f0 + amplitudes, and utterances are independent: the drivers run such kernels side by
// side on an internal side stream and join it on the caller's stream before returning (event record / wait only: no
// host synchronisation, legal under stream capture).  Streams and events are cached per host thread and device
// (thread_local: two threads calling into the library never share an event, so one thread's record can never be
// picked up by the other's wait).
//   mode 0: everything on the caller's stream, in order
//   mode 1: impulse responses on a high-priority side stream next to the bank / comb source
//   mode k >= 2: additionally the batch is cut into k sub-batches that alternate between the caller's stream and the
//           side stream, staggered (the side stream starts with the impulse responses of the WHOLE batch), so the
//           FIR of one sub-batch (shared-memory / latency bound) shares the SMs with the bank of the next (FMA / SFU
//           bound).  Results do not depend on the mode: the noise is keyed by the global utterance index and the
//           FFT-domain FIR is bit-identical for any batch split.
//   mode -k: as k, with the high-priority stream as the side stream
// ---------------------------------------------------------------------------------------
namespace b2d {
std::atomic<int> g_overlap{1};

struct SideLane {
    cudaStream_t hi = nullptr, lo = nullptr;       // high- and normal-priority side streams
    cudaEvent_t ev = nullptr;                      // every record is waited on right away (SideFork)
    bool ok = false;
};
struct SideLanes {
    SideLane lane[64];
    ~SideLanes() {
        for (SideLane& l : lane) {
            if (l.ev) cudaEventDestroy(l.ev);
            if (l.hi) cudaStreamDestroy(l.hi);        // deferred by the runtime until queued work has drained
            if (l.lo) cudaStreamDestroy(l.lo);
        }
    }
};

// nullptr = run everything on the caller's stream (mode 0, or the streams could not be created)
static SideLane* side_lane() {
    static thread_local SideLanes lanes;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    SideLane& l = lanes.lane[dev];
    if (!l.ok) {
        if (l.hi) return nullptr;                        // creation failed before: do not retry on every call
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);      // hi = numerically lowest = greatest priority
        bool good = cudaStreamCreateWithPriority(&l.hi, cudaStreamNonBlocking, hi) == cudaSuccess;
        good = good && cudaStreamCreateWithFlags(&l.lo, cudaStreamNonBlocking) == cudaSuccess;
        good = good && cudaEventCreateWithFlags(&l.ev, cudaEventDisableTiming) == cudaSuccess;
        if (!good) { cudaGetLastError(); if (!l.hi) l.hi = (cudaStream_t)1; return nullptr; }
        l.ok = true;
    }
    return &l;
}

// The side streams of one driver call on the caller's stream `st`.  fork() starts side streams after the work enqueued
// so far on `st`; wait_side() makes `st` wait for the work enqueued so far on every forked side stream.  After fork(),
// every exit path goes through join(), also after a failed launch: a side stream that `st` does not wait for leaves
// work behind the caller's back and makes a stream capture end with an error.  join() returns the first error: the
// launch error it is given, else the first failed event record / wait.  A stream never waits for itself, so without a
// lane (hi() == lo() == st) no event is touched.
class SideFork {
public:
    SideFork(SideLane* lane, cudaStream_t st, const char* who) : lane_(lane), st_(st), who_(who) {}
    cudaStream_t hi() const { return lane_ ? lane_->hi : st_; }
    cudaStream_t lo() const { return lane_ ? lane_->lo : st_; }
    bool ok() const { return err_ == cudaSuccess; }

    bool fork(cudaStream_t a, cudaStream_t b) {
        if (a == st_ && b == st_) return true;
        if (!note(cudaEventRecord(lane_->ev, st_), "fork")) return false;
        for (cudaStream_t q : {a, b}) {
            if (q == st_ || (n_ == 1 && side_[0] == q)) continue;
            if (!note(cudaStreamWaitEvent(q, lane_->ev, 0), "fork")) return false;
            side_[n_++] = q;
        }
        return true;
    }
    void wait_side(const char* what = "event") {
        for (int i = 0; i < n_; ++i) {
            cudaError_t e = cudaEventRecord(lane_->ev, side_[i]);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(st_, lane_->ev, 0);
            note(e, what);
        }
    }
    int join(int rc) {
        wait_side("join");
        if (rc) return rc;
        if (!ok()) return fail((int)err_, "%s: %s: %s", who_, what_, cudaGetErrorString(err_));
        return 0;
    }

private:
    bool note(cudaError_t e, const char* what) {
        if (e != cudaSuccess && ok()) { err_ = e; what_ = what; }
        return e == cudaSuccess;
    }
    SideLane* lane_;
    cudaStream_t st_;
    const char* who_;
    cudaStream_t side_[2] = {};
    int n_ = 0;
    cudaError_t err_ = cudaSuccess;
    const char* what_ = "";
};
}  // namespace b2d

// 0 = auto = 1 (separate bank kernel), 1 = separate bank kernel, 2 = bank fused into the FFT-domain FIR kernel: with 168
// registers only three 4-warp CTAs fit an SM, and ONE warp per scheduler in the bank phase cannot keep the FMA pipe busy
// (the stand-alone bank kernel has four).  It stays selectable: one launch less, no [B, T] sinusoid round trip.
namespace b2d { std::atomic<int> g_sins_impl{0}; }
extern "C" int b2d_set_sins_impl(int impl) {
    if (impl < 0 || impl > 3) return b2d::fail(B2D_ERR_UNSUPPORTED, "set_sins_impl: %d not in {0, 1, 2, 3}", impl);
    b2d::g_sins_impl.store(impl, std::memory_order_relaxed);
    return 0;
}

extern "C" int b2d_set_overlap(int mode) {
    if (mode < -64 || mode > 64) return b2d::fail(B2D_ERR_UNSUPPORTED, "set_overlap: %d outside [-64, 64]", mode);
    b2d::g_overlap.store(mode, std::memory_order_relaxed);
    return 0;
}

extern "C" int b2d_set_fft_arith(int packed) {
    if (packed != 0 && packed != 1) return b2d::fail(B2D_ERR_UNSUPPORTED, "set_fft_arith: %d not in {0, 1}", packed);
    b2d::g_fft_packed.store(packed, std::memory_order_relaxed);
    return 0;
}

extern "C" int b2d_version(void) { return B2D_VERSION; }
extern "C" const char* b2d_last_error(void) { return b2d::err_buf(); }

// ---------------------------------------------------------------------------------------
// Sins: bank -> all-pass IR -> noise IR -> two FIRs + mix        (ddsp/vocoder.py:580-611)
// workspace: b2d::sins_workspace (b2d_common.cuh)
// ---------------------------------------------------------------------------------------
// the spectrum buffers exist under b2d_set_sins_impl(3), for the shapes the spectrum kernels take
static bool sins_spectra(int impl, int block, int n_mag_allpass, int n_mag_noise) {
    return impl == 3 && b2d::fir_spec_supported(block, 2 * (n_mag_allpass - 1), 2 * (n_mag_noise - 1));
}

extern "C" size_t b2d_sins_workspace_bytes(int B, int n_frames, int block, int n_mag_allpass, int n_mag_noise) {
    const int impl = b2d::g_sins_impl.load(std::memory_order_relaxed);
    return b2d::sins_workspace(B, n_frames, block, n_mag_allpass, n_mag_noise,
                               sins_spectra(impl, block, n_mag_allpass, n_mag_noise)).bytes;
}

extern "C" int b2d_sins_synth(const float* f0_frames, const double* frame_phase, const float* c_amp,
                              const float* c_group_delay, const float* c_noise, int64_t ctrl_stride,
                              const float* noise_in, uint64_t seed, int64_t utterance_offset,
                              const float* dft_tables_allpass, const float* dft_tables_noise, int B, int n_frames,
                              int block, int n_harmonics, int n_mag_allpass, int n_mag_noise,
                              double sampling_rate, int round_fp32, float* signal, float* harmonic,
                              float* noise_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!workspace) return b2d::fail(B2D_ERR_NULL, "sins_synth: null workspace");
    const int impl = b2d::g_sins_impl.load(std::memory_order_relaxed);
    const b2d::SinsWorkspace w = b2d::sins_workspace(B, n_frames, block, n_mag_allpass, n_mag_noise,
                                                     sins_spectra(impl, block, n_mag_allpass, n_mag_noise));
    if (w.bytes == 0) return b2d::fail(B2D_ERR_SHAPE, "sins_synth: bad shape");
    if (workspace_bytes < w.bytes) return b2d::fail(B2D_ERR_WORKSPACE, "sins_synth: workspace %zu < %zu bytes", workspace_bytes, w.bytes);
    if ((reinterpret_cast<uintptr_t>(workspace) & 255u) != 0) return b2d::fail(B2D_ERR_ALIGN, "sins_synth: workspace must be 256-byte aligned");
    const int La = 2 * (n_mag_allpass - 1), Ln = 2 * (n_mag_noise - 1);
    float* sinus = b2d::ws_at(workspace, w.sinus);
    float* ir_ap = b2d::ws_at(workspace, w.ir_ap);
    float* ir_n = b2d::ws_at(workspace, w.ir_n);

    if (block % 256 != 0)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_synth: block size %d must be a multiple of 256", block);
    if (La != Ln && !noise_out) return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_synth: noise_out required when n_mag_allpass != n_mag_noise");
    cudaStream_t st = (cudaStream_t)stream;
    const int mode = b2d::g_overlap.load(std::memory_order_relaxed);
    b2d::SideLane* lane = mode != 0 ? b2d::side_lane() : nullptr;
    int nsplit = (mode < 0 ? -mode : mode);
    if (nsplit < 2 || !lane) nsplit = 1;
    if (nsplit > B) nsplit = B;
    b2d::SideFork f(lane, st, "sins_synth");

    // one sub-batch [b0, b0 + nb): bank, then (after the impulse responses) the FIRs, all on stream `q`
    auto bank = [&](int b0, int nb, cudaStream_t q) -> int {
        return b2d_sins_bank(f0_frames + (size_t)b0 * n_frames, frame_phase + (size_t)b0 * n_frames,
                             c_amp + (size_t)b0 * n_frames * ctrl_stride, ctrl_stride, nb, n_frames, block, n_harmonics,
                             sampling_rate, round_fp32, sinus + (size_t)b0 * n_frames * block, q);
    };
    auto firs = [&](int b0, int nb, cudaStream_t q) -> int {
        const size_t ot = (size_t)b0 * n_frames * block, of = (size_t)b0 * n_frames;
        const float* nz_in = noise_in ? noise_in + ot : nullptr;
        float* harm = harmonic ? harmonic + ot : nullptr;
        float* nz_out = noise_out ? noise_out + ot : nullptr;
        if (La == Ln)
            return b2d::ltv_fir_launch(sinus + ot, ir_ap + of * La, La, harm, nz_in, ir_n + of * Ln, Ln, nz_out, nullptr,
                                       signal + ot, seed, utterance_offset + b0, nb, n_frames, block, q);
        // different tap counts: two launches, the second adds the first's output
        int r = b2d::ltv_fir_launch(nz_in, ir_n + of * Ln, Ln, nz_out, nullptr, nullptr, 0, nullptr, nullptr, nullptr, seed,
                                    utterance_offset + b0, nb, n_frames, block, q);
        if (r) return r;
        return b2d::ltv_fir_launch(sinus + ot, ir_ap + of * La, La, harm, nullptr, nullptr, 0, nullptr, nz_out, signal + ot,
                                   seed, utterance_offset + b0, nb, n_frames, block, q);
    };
    auto irs = [&](cudaStream_t q, cudaStream_t q2) -> int {
        int r = b2d_ir_build(c_group_delay, ctrl_stride, B2D_IR_ALLPASS, nullptr, dft_tables_allpass, B, n_frames,
                             n_mag_allpass, sampling_rate, ir_ap, q);
        if (r) return r;
        return b2d_ir_build(c_noise, ctrl_stride, B2D_IR_MAG_HANN, nullptr, dft_tables_noise, B, n_frames, n_mag_noise,
                            sampling_rate, ir_n, q2);
    };
    // ---- spectrum path (opt-in, b2d_set_sins_impl(3)): impulse responses -> their packed spectra once per frame (both on
    // the side stream, beside the bank), then the FIR kernel reads the spectra: a quarter of its transforms and a third of
    // its shared memory disappear (126 registers, 53 KB: 4 CTAs per SM instead of 3).  The transform of the impulse
    // responses is only MOVED and the FIR kernel waits for the spectra right before its products; it pays only once the
    // tensor-core GEMM of the impulse-response stage emits these spectra itself.  Kept as the tested consumer side of that
    // plan. ----
    if (impl == 3 && !(b2d::fir_spec_supported(block, La, Ln) && b2d::fir_fft_selected()))
        return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_synth: spectrum path needs block 512, <= 512 taps and the FFT-domain FIR");
    if (impl == 3) {
        float* spec_ap = b2d::ws_at(workspace, w.spec_ap);
        float* spec_n = b2d::ws_at(workspace, w.spec_n);
        const cudaStream_t q = f.hi();
        int rc = 0;
        if (f.fork(q, q)) {
            rc = irs(q, q);
            if (!rc) rc = b2d::ir_spectrum_launch(ir_ap, La, spec_ap, ir_n, Ln, spec_n, B, n_frames, q);
            if (!rc) rc = bank(0, B, st);
        }
        rc = f.join(rc);
        if (rc) return rc;
        return b2d::ltv_fir_fft_spec_launch(sinus, spec_ap, La, harmonic, noise_in, spec_n, Ln, noise_out, signal, seed,
                                            utterance_offset, B, n_frames, block, st);
    }
    // ---- fused path: impulse responses (side by side on the two side streams), then ONE kernel: bank + both FIRs + mix ----
    if (impl == 2 && !(b2d::sins_fused_supported(block, La, Ln, n_harmonics) && b2d::fir_fft_selected()))
        return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_synth: fused kernel needs block 512, <= 512 taps, <= 128 harmonics and the FFT-domain FIR");
    if (impl == 2) {
        const int rc = f.join(f.fork(f.hi(), f.lo()) ? irs(f.hi(), f.lo()) : 0);
        if (rc) return rc;
        return b2d::sins_fused_launch(f0_frames, frame_phase, c_amp, ctrl_stride, n_harmonics, sampling_rate, round_fp32,
                                      ir_ap, La, harmonic, noise_in, ir_n, Ln, noise_out, signal, seed, utterance_offset,
                                      B, n_frames, block, st);
    }
    // the side stream starts with the impulse responses of the whole batch (launched first: one 512-thread CTA per SM,
    // latency bound), the caller's stream with the first bank.  A small launch (one utterance, one pipeline chunk)
    // leaves most SMs idle: its two impulse-response builds are latency bound single waves, so they run side by side on
    // the two side streams instead of one after the other.
    const cudaStream_t side = (mode == 1 || mode < 0) ? f.hi() : f.lo();
    const bool two_lanes = lane && nsplit == 1 && (long long)B * n_frames <= (long long)b2d::num_sms() * 64;
    const cudaStream_t side2 = two_lanes ? (side == f.hi() ? f.lo() : f.hi()) : side;
    int rc = f.fork(side, side2) ? irs(side, side2) : 0;
    for (int s = 0; s < nsplit && !rc && f.ok(); ++s) {
        const int b0 = (int)((long long)B * s / nsplit), b1 = (int)((long long)B * (s + 1) / nsplit);
        const cudaStream_t q = (s & 1) ? side : st;
        rc = bank(b0, b1 - b0, q);
        if (s == 0) f.wait_side();          // the impulse responses, before the first FIR on the caller's stream
        if (!rc && f.ok()) rc = firs(b0, b1 - b0, q);
    }
    return f.join(rc);
}

// ---------------------------------------------------------------------------------------
// CombSub (old): comb source -> all-pass FIR -> dynamic-window harmonic FIR, + noise FIR
// (ddsp/vocoder.py:834-862).
// workspace: b2d::combsub_workspace (b2d_common.cuh)
// ---------------------------------------------------------------------------------------
extern "C" int b2d_comb_source(const float*, const double*, int, int, int, double, int, float*, void*);

extern "C" size_t b2d_combsub_workspace_bytes(int B, int n_frames, int block, int n_mag_allpass,
                                              int n_mag_harmonic, int n_mag_noise) {
    return b2d::combsub_workspace(B, n_frames, block, n_mag_allpass, n_mag_harmonic, n_mag_noise).bytes;
}

extern "C" int b2d_combsub_synth(const float* f0_frames, const double* frame_phase, const float* c_group_delay,
                                 const float* c_harmonic, const float* c_noise, int64_t ctrl_stride,
                                 const float* noise_in, uint64_t seed, int64_t utterance_offset,
                                 const float* dft_tables_allpass, const float* dft_tables_harmonic,
                                 const float* dft_tables_noise, int B, int n_frames, int block,
                                 int n_mag_allpass, int n_mag_harmonic, int n_mag_noise, double sampling_rate,
                                 int round_fp32, float* signal, float* harmonic, float* noise_out, void* workspace,
                                 size_t workspace_bytes, void* stream) {
    if (!workspace) return b2d::fail(B2D_ERR_NULL, "combsub_synth: null workspace");
    const b2d::CombSubWorkspace w = b2d::combsub_workspace(B, n_frames, block, n_mag_allpass, n_mag_harmonic, n_mag_noise);
    if (w.bytes == 0) return b2d::fail(B2D_ERR_SHAPE, "combsub_synth: bad shape");
    if (workspace_bytes < w.bytes) return b2d::fail(B2D_ERR_WORKSPACE, "combsub_synth: workspace %zu < %zu bytes", workspace_bytes, w.bytes);
    if ((reinterpret_cast<uintptr_t>(workspace) & 255u) != 0) return b2d::fail(B2D_ERR_ALIGN, "combsub_synth: workspace must be 256-byte aligned");
    if (block % 256 != 0) return b2d::fail(B2D_ERR_UNSUPPORTED, "combsub_synth: block size %d must be a multiple of 256", block);
    const int La = 2 * (n_mag_allpass - 1), Lh = 2 * (n_mag_harmonic - 1), Ln = 2 * (n_mag_noise - 1);
    float* comb = b2d::ws_at(workspace, w.comb);
    float* allp = b2d::ws_at(workspace, w.allpassed);
    float* nbuf = noise_out ? noise_out : b2d::ws_at(workspace, w.noise);
    float* ir_ap = b2d::ws_at(workspace, w.ir_ap);
    float* ir_h = b2d::ws_at(workspace, w.ir_h);
    float* ir_n = b2d::ws_at(workspace, w.ir_n);
    cudaStream_t st = (cudaStream_t)stream;

    // comb source -> all-pass filter, and the noise filter, on the caller's stream
    auto front = [&]() -> int {
        int r = b2d_comb_source(f0_frames, frame_phase, B, n_frames, block, sampling_rate, round_fp32, comb, stream);
        if (!r) r = b2d_ir_build(c_group_delay, ctrl_stride, B2D_IR_ALLPASS, nullptr, dft_tables_allpass, B, n_frames,
                                 n_mag_allpass, sampling_rate, ir_ap, stream);
        if (!r) r = b2d_ir_build(c_noise, ctrl_stride, B2D_IR_MAG_HANN, nullptr, dft_tables_noise, B, n_frames, n_mag_noise,
                                 sampling_rate, ir_n, stream);
        if (r) return r;
        // all-pass on the comb and the noise filter: one launch when the tap counts agree
        if (La == Ln)
            return b2d::ltv_fir_launch(comb, ir_ap, La, allp, noise_in, ir_n, Ln, nbuf, nullptr, nullptr, seed,
                                       utterance_offset, B, n_frames, block, st);
        r = b2d::ltv_fir_launch(comb, ir_ap, La, allp, nullptr, nullptr, 0, nullptr, nullptr, nullptr, seed,
                                utterance_offset, B, n_frames, block, st);
        if (r) return r;
        return b2d::ltv_fir_launch(noise_in, ir_n, Ln, nbuf, nullptr, nullptr, 0, nullptr, nullptr, nullptr, seed,
                                   utterance_offset, B, n_frames, block, st);
    };
    // the dynamic-window impulse response (the largest of the three builds) is only needed by the LAST filter: it runs
    // on the internal side stream beside the front and is joined right before the harmonic filter
    b2d::SideLane* lane = b2d::g_overlap.load(std::memory_order_relaxed) != 0 ? b2d::side_lane() : nullptr;
    b2d::SideFork f(lane, st, "combsub_synth");
    const cudaStream_t q = f.hi();
    int rc = 0;
    if (f.fork(q, q)) {
        const int rch = b2d_ir_build(c_harmonic, ctrl_stride, B2D_IR_MAG_DYNAMIC, f0_frames, dft_tables_harmonic, B,
                                     n_frames, n_mag_harmonic, sampling_rate, ir_h, q);
        rc = front();
        if (!rc) rc = rch;
    }
    rc = f.join(rc);
    if (rc) return rc;
    // harmonic magnitude filter on the all-passed comb; signal = harmonic + noise
    return b2d::ltv_fir_launch(allp, ir_h, Lh, harmonic, nullptr, nullptr, 0, nullptr, nbuf, signal, seed,
                               utterance_offset, B, n_frames, block, st);
}

// ---------------------------------------------------------------------------------------
// NSF-HiFiGAN generator (nsf_hifigan/models.py:207-273): the kernels of hifigan.cu
// ---------------------------------------------------------------------------------------
namespace b2d {
int hifigan_conv_launch(const float* x, int64_t sb, int64_t st, int64_t sc, int B, int T, int Cin, const float* w,
                        const float* bias, int k, int dil, int N, int lrelu, const float* residual, const float* accum,
                        float div, int up, const float* src, const float* wn, const float* bn, int n_k, int n_stride,
                        int n_pad, float* out, cudaStream_t stream);
int hifigan_post_launch(const float* x, const float* w, const float* bias, int B, int T, int C, float* out, cudaStream_t stream);
}  // namespace b2d

extern "C" int b2d_hifigan_conv(const float* x, int64_t x_stride_b, int64_t x_stride_t, int64_t x_stride_c, int B, int T,
                                int C_in, const float* w, const float* bias, int k, int dilation, int N, int lrelu,
                                const float* residual, const float* accum, float div, int up, const float* source,
                                const float* noise_w, const float* noise_b, int noise_k, int noise_stride, int noise_pad,
                                float* out, void* stream) {
    if (!x || !w || !bias || !out || (source && (!noise_w || !noise_b)))
        return b2d::fail(B2D_ERR_NULL, "hifigan_conv: null pointer");
    if (B <= 0 || T <= 0 || C_in <= 0 || N <= 0 || k <= 0 || dilation <= 0 || !(div > 0.f) || up < 0 ||
        (up && N % up) || (source && (noise_k <= 0 || noise_stride <= 0 || noise_pad < 0)))
        return b2d::fail(B2D_ERR_SHAPE, "hifigan_conv: bad shape");
    if (k % 2 == 0 || C_in % 16 || N % 16 || (up && ((N / up) % 2 || residual || accum)) || (!up && source) ||
        B > 65535 || (long long)dilation * (k - 1) / 2 > 256)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "hifigan_conv: needs odd k, a halo of <= 256 rows, C_in and N multiples of "
                                              "16, an even C_out, no residual / accum with up, no source without");
    if (x_stride_c == 1 && (!b2d::aligned16(x) || x_stride_t % 4 || x_stride_b % 4))
        return b2d::fail(B2D_ERR_ALIGN, "hifigan_conv: a unit channel stride needs 16-byte aligned x and strides");
    if (!b2d::aligned16(w) || (reinterpret_cast<uintptr_t>(bias) & 7u) || (reinterpret_cast<uintptr_t>(out) & 7u) ||
        (residual && (reinterpret_cast<uintptr_t>(residual) & 7u)) || (accum && (reinterpret_cast<uintptr_t>(accum) & 7u)))
        return b2d::fail(B2D_ERR_ALIGN, "hifigan_conv: w 16-byte, bias / out / residual / accum 8-byte aligned");
    return b2d::hifigan_conv_launch(x, x_stride_b, x_stride_t, x_stride_c, B, T, C_in, w, bias, k, dilation, N, lrelu,
                                    residual, accum, div, up, source, noise_w, noise_b, noise_k, noise_stride, noise_pad,
                                    out, (cudaStream_t)stream);
}

extern "C" int b2d_hifigan_post(const float* x, const float* w, const float* bias, int B, int T, int C, float* out, void* stream) {
    if (!x || !w || !bias || !out) return b2d::fail(B2D_ERR_NULL, "hifigan_post: null pointer");
    if (B <= 0 || T <= 0 || C <= 0) return b2d::fail(B2D_ERR_SHAPE, "hifigan_post: bad shape");
    if (C % 4 || C > 4096) return b2d::fail(B2D_ERR_UNSUPPORTED, "hifigan_post: C must be a multiple of 4, <= 4096");
    if (!b2d::aligned16(x)) return b2d::fail(B2D_ERR_ALIGN, "hifigan_post: x must be 16-byte aligned");
    return b2d::hifigan_post_launch(x, w, bias, B, T, C, out, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// RMVPE pitch extractor (encoder/rmvpe/), inference: the kernels of rmvpe.cu
// ---------------------------------------------------------------------------------------------------------------------
namespace b2d {
int rmvpe_conv_launch(const float* x, int ldx, int B, int T, int F, int Cin, const float* w, const float* bias, int k,
                      int N, int n_valid, int act, int up, const float* res, int ldr, float* out, int ldo,
                      cudaStream_t stream);
int rmvpe_conv_small_launch(const float* x, int64_t sb, int64_t st, int64_t sf, int64_t sc, int B, int T, int F, int Cin,
                            const float* in_scale, const float* in_shift, const float* w, const float* bias, int k,
                            int Cout, int act, int head, float* out, int ldo, cudaStream_t stream);
int rmvpe_pool_launch(const float* x, int ldx, int B, int T, int F, int C, float* out, cudaStream_t stream);
int rmvpe_gru_launch(const float* xg, const float* whh, const float* bhh, int B, int T, float* out, cudaStream_t stream);
int rmvpe_resample_launch(const float* x, int B, int N, const float* table, int new_freq, int orig_freq, int taps,
                          int width, int n_out, float* out, cudaStream_t stream);
int rmvpe_mel_launch(const float* y, int B, int N, const float* window, const float* basis, const int* lohi, int hop,
                     int n_frames, int t_pad, float* out, cudaStream_t stream);
int rmvpe_decode_launch(const float* sal, int B, int t_pad, int n_frames, float thred, float* f0, cudaStream_t stream);
}  // namespace b2d

namespace {
bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }
bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }
}  // namespace

extern "C" int b2d_rmvpe_conv(const float* x, int ldx, int B, int T, int F, int C_in, const float* w, const float* bias,
                              int k, int N, int n_valid, int act, int up, const float* residual, int ldr, float* out,
                              int ldo, void* stream) {
    if (!x || !w || !bias || !out) return b2d::fail(B2D_ERR_NULL, "rmvpe_conv: null pointer");
    if (B <= 0 || T <= 0 || F <= 0 || C_in <= 0 || N <= 0 || n_valid <= 0 || n_valid > N || ldx < C_in ||
        ldo < (up ? N / 4 : n_valid) || (residual && ldr < n_valid) || act < 0 || act > 2)
        return b2d::fail(B2D_ERR_SHAPE, "rmvpe_conv: bad shape");
    if (k < 1 || k > 3 || C_in % 16 || N % 16 || n_valid % 2 || !pow2(F) || B > 65535 || N / 16 > 65535 ||
        (up && (k != 2 || N % 8 || n_valid != N || residual)))
        return b2d::fail(B2D_ERR_UNSUPPORTED, "rmvpe_conv: needs k in 1..3, C_in and N multiples of 16, an even n_valid, "
                                              "F a power of two; up needs k = 2, N = 4 C_out with C_out even, no residual");
    if (!b2d::aligned16(x) || ldx % 4 || !b2d::aligned16(w) || !aligned8(bias) || !aligned8(out) || ldo % 2 ||
        (residual && (!aligned8(residual) || ldr % 2)))
        return b2d::fail(B2D_ERR_ALIGN, "rmvpe_conv: x / w 16-byte aligned with ldx % 4 == 0; bias / out / residual "
                                        "8-byte aligned with even strides");
    return b2d::rmvpe_conv_launch(x, ldx, B, T, F, C_in, w, bias, k, N, n_valid, act, up, residual, ldr, out, ldo,
                                  (cudaStream_t)stream);
}

extern "C" int b2d_rmvpe_conv_small(const float* x, int64_t x_stride_b, int64_t x_stride_t, int64_t x_stride_f,
                                    int64_t x_stride_c, int B, int T, int F, int C_in, const float* in_scale,
                                    const float* in_shift, const float* w, const float* bias, int k, int C_out, int relu,
                                    int head, float* out, int ldo, void* stream) {
    if (!x || !w || !out || (!in_scale != !in_shift)) return b2d::fail(B2D_ERR_NULL, "rmvpe_conv_small: null pointer");
    if (B <= 0 || T <= 0 || F <= 0 || C_in <= 0 || C_out <= 0 || (!head && ldo < C_out))
        return b2d::fail(B2D_ERR_SHAPE, "rmvpe_conv_small: bad shape");
    if ((k != 1 && k != 3) || C_out > 16 || C_in * C_out * k * k > 4096)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "rmvpe_conv_small: k 1 or 3, C_out <= 16, C_in C_out k^2 <= 4096");
    return b2d::rmvpe_conv_small_launch(x, x_stride_b, x_stride_t, x_stride_f, x_stride_c, B, T, F, C_in, in_scale,
                                        in_shift, w, bias, k, C_out, relu, head, out, ldo, (cudaStream_t)stream);
}

extern "C" int b2d_rmvpe_pool(const float* x, int ldx, int B, int T, int F, int C, float* out, void* stream) {
    if (!x || !out) return b2d::fail(B2D_ERR_NULL, "rmvpe_pool: null pointer");
    if (B <= 0 || T <= 0 || F <= 0 || C <= 0 || ldx < C || T % 2 || F % 2)
        return b2d::fail(B2D_ERR_SHAPE, "rmvpe_pool: bad shape (T and F must be even)");
    return b2d::rmvpe_pool_launch(x, ldx, B, T, F, C, out, (cudaStream_t)stream);
}

extern "C" int b2d_rmvpe_gru(const float* xg, const float* w_hh, const float* b_hh, int B, int T, float* out,
                             void* stream) {
    if (!xg || !w_hh || !b_hh || !out) return b2d::fail(B2D_ERR_NULL, "rmvpe_gru: null pointer");
    if (B <= 0 || T <= 0 || B > 4 * 65535) return b2d::fail(B2D_ERR_SHAPE, "rmvpe_gru: bad shape");
    return b2d::rmvpe_gru_launch(xg, w_hh, b_hh, B, T, out, (cudaStream_t)stream);
}

extern "C" int b2d_rmvpe_resample(const float* x, int B, int N, const float* table, int new_freq, int orig_freq,
                                  int taps, int width, int n_out, float* out, void* stream) {
    if (!x || !table || !out) return b2d::fail(B2D_ERR_NULL, "rmvpe_resample: null pointer");
    if (B <= 0 || N <= 0 || new_freq <= 0 || orig_freq <= 0 || taps <= 0 || width < 0 || n_out <= 0)
        return b2d::fail(B2D_ERR_SHAPE, "rmvpe_resample: bad shape");
    return b2d::rmvpe_resample_launch(x, B, N, table, new_freq, orig_freq, taps, width, n_out, out, (cudaStream_t)stream);
}

extern "C" int b2d_rmvpe_mel(const float* audio, int B, int N, const float* window, const float* basis, const int* lohi,
                             int hop, int n_frames, int t_pad, float* out, void* stream) {
    if (!audio || !window || !basis || !lohi || !out) return b2d::fail(B2D_ERR_NULL, "rmvpe_mel: null pointer");
    if (B <= 0 || B > 65535 || hop <= 0 || n_frames <= 0 || t_pad < n_frames)
        return b2d::fail(B2D_ERR_SHAPE, "rmvpe_mel: bad shape");
    if (N <= 512 || n_frames != 1 + N / hop)
        return b2d::fail(B2D_ERR_SHAPE, "rmvpe_mel: needs N > 512 samples (reflect padding) and n_frames = 1 + N / hop");
    return b2d::rmvpe_mel_launch(audio, B, N, window, basis, lohi, hop, n_frames, t_pad, out, (cudaStream_t)stream);
}

extern "C" int b2d_rmvpe_decode(const float* salience, int B, int t_pad, int n_frames, float thred, float* f0,
                                void* stream) {
    if (!salience || !f0) return b2d::fail(B2D_ERR_NULL, "rmvpe_decode: null pointer");
    if (B <= 0 || n_frames <= 0 || t_pad < n_frames) return b2d::fail(B2D_ERR_SHAPE, "rmvpe_decode: bad shape");
    return b2d::rmvpe_decode_launch(salience, B, t_pad, n_frames, thred, f0, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// HuBERT / ContentVec units encoder, inference: the kernels of hubert.cu
// ---------------------------------------------------------------------------------------------------------------------
namespace b2d {
int hubert_conv0_launch(const float* x, int B, int N, int pad, const float* w, int L0, int La, float* y, double* part,
                        cudaStream_t stream);
int hubert_gn_finalize_launch(const double* part, int B, int n_tiles, int L0, const float* gamma, const float* beta,
                              float eps, float* scale, float* shift, cudaStream_t stream);
int hubert_act_launch(const float* x, int rows, int C, int rows_per_b, const float* scale, const float* shift, float* hi,
                      float* lo, cudaStream_t stream);
int hubert_ln_launch(const float* x, const float* y, int rows, int T, int rows_per_b, int C, int gelu,
                     const float* gamma, const float* beta, float eps, float* h, float* hi, float* lo,
                     cudaStream_t stream);
int hubert_posconv_launch(const float* x, int B, int T, const float* w, const float* bias, float* y,
                          cudaStream_t stream);
int hubert_attention_launch(const float* qkv, int B, int T, float* hi, float* lo, cudaStream_t stream);
int hubert_align_launch(const float* units, int B, int T, int C, float ratio, int n_frames, float* out,
                        cudaStream_t stream);
}  // namespace b2d

extern "C" int b2d_hubert_conv0(const float* x, int B, int N, int pad, const float* w, int La, float* y, double* part,
                                void* stream) {
    if (!x || !w || !y || !part) return b2d::fail(B2D_ERR_NULL, "hubert_conv0: null pointer");
    if (B <= 0 || B > 65535 || N <= 0 || pad < 0 || (long long)N + 2LL * pad < 10)
        return b2d::fail(B2D_ERR_SHAPE, "hubert_conv0: bad shape (N + 2 pad must be >= 10)");
    const int L0 = (N + 2 * pad - 10) / 5 + 1;
    if (La < L0) return b2d::fail(B2D_ERR_SHAPE, "hubert_conv0: La %d < L0 %d", La, L0);
    return b2d::hubert_conv0_launch(x, B, N, pad, w, L0, La, y, part, (cudaStream_t)stream);
}

extern "C" int b2d_hubert_gn_finalize(const double* part, int B, int n_tiles, int L0, const float* gamma,
                                      const float* beta, float eps, float* scale, float* shift, void* stream) {
    if (!part || !gamma || !beta || !scale || !shift) return b2d::fail(B2D_ERR_NULL, "hubert_gn_finalize: null pointer");
    if (B <= 0 || n_tiles <= 0 || L0 <= 0 || L0 > 64LL * n_tiles || !(eps > 0.f))
        return b2d::fail(B2D_ERR_SHAPE, "hubert_gn_finalize: bad shape");
    return b2d::hubert_gn_finalize_launch(part, B, n_tiles, L0, gamma, beta, eps, scale, shift, (cudaStream_t)stream);
}

extern "C" int b2d_hubert_act(const float* x, int rows, int C, int rows_per_b, const float* scale, const float* shift,
                              float* hi, float* lo, void* stream) {
    if (!x || !hi || (scale && !shift) || (shift && !scale)) return b2d::fail(B2D_ERR_NULL, "hubert_act: null pointer");
    if (rows <= 0 || C <= 0 || rows_per_b <= 0 || rows % rows_per_b)
        return b2d::fail(B2D_ERR_SHAPE, "hubert_act: bad shape (rows must be a multiple of rows_per_b)");
    return b2d::hubert_act_launch(x, rows, C, rows_per_b, scale, shift, hi, lo, (cudaStream_t)stream);
}

extern "C" int b2d_hubert_ln(const float* x, const float* y, int rows, int T, int rows_per_b, int C, int gelu,
                             const float* gamma, const float* beta, float eps, float* h, float* hi, float* lo,
                             void* stream) {
    if (!x || !gamma || !beta || (!h && !hi) || (lo && !hi)) return b2d::fail(B2D_ERR_NULL, "hubert_ln: null pointer");
    if (rows <= 0 || T <= 0 || rows % T || rows_per_b < T || !(eps > 0.f))
        return b2d::fail(B2D_ERR_SHAPE, "hubert_ln: bad shape");
    if (C != 512 && C != 768) return b2d::fail(B2D_ERR_UNSUPPORTED, "hubert_ln: C must be 512 or 768, got %d", C);
    if (h == x && rows_per_b != T) return b2d::fail(B2D_ERR_SHAPE, "hubert_ln: h may alias x only when rows_per_b = T");
    return b2d::hubert_ln_launch(x, y, rows, T, rows_per_b, C, gelu, gamma, beta, eps, h, hi, lo, (cudaStream_t)stream);
}

extern "C" int b2d_hubert_posconv(const float* x, int B, int T, const float* w, const float* bias, float* y,
                                  void* stream) {
    if (!x || !w || !bias || !y) return b2d::fail(B2D_ERR_NULL, "hubert_posconv: null pointer");
    if (B <= 0 || B > 65535 || T <= 0) return b2d::fail(B2D_ERR_SHAPE, "hubert_posconv: bad shape");
    if (!b2d::aligned16(w)) return b2d::fail(B2D_ERR_ALIGN, "hubert_posconv: w must be 16-byte aligned");
    return b2d::hubert_posconv_launch(x, B, T, w, bias, y, (cudaStream_t)stream);
}

extern "C" int b2d_hubert_attention(const float* qkv, int B, int T, float* hi, float* lo, void* stream) {
    if (!qkv || !hi) return b2d::fail(B2D_ERR_NULL, "hubert_attention: null pointer");
    if (B <= 0 || B > 65535 || T <= 0) return b2d::fail(B2D_ERR_SHAPE, "hubert_attention: bad shape");
    return b2d::hubert_attention_launch(qkv, B, T, hi, lo, (cudaStream_t)stream);
}

extern "C" int b2d_hubert_align(const float* units, int B, int T, int C, float ratio, int n_frames, float* out,
                                void* stream) {
    if (!units || !out) return b2d::fail(B2D_ERR_NULL, "hubert_align: null pointer");
    if (B <= 0 || T <= 0 || C <= 0 || n_frames <= 0 || !(ratio >= 0.f) || !(ratio < 1e30f))
        return b2d::fail(B2D_ERR_SHAPE, "hubert_align: bad shape");
    return b2d::hubert_align_launch(units, B, T, C, ratio, n_frames, out, (cudaStream_t)stream);
}
