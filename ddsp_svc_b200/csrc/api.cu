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
