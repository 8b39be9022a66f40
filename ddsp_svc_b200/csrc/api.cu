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
size_t fir_spec_floats(int B, int nF);
int ir_spectrum_launch(const float* ir1, int taps1, float* spec1, const float* ir2, int taps2, float* spec2, int B, int nF,
                       cudaStream_t st);
int ltv_fir_fft_spec_launch(const float* x1, const float* spec1, int taps1, float* y1, const float* x2, const float* spec2,
                            int taps2, float* y2, float* mix, uint64_t seed, int64_t utt_off, int B, int nF, int P, cudaStream_t st);
bool sins_fused_supported(int P, int taps_allpass, int taps_noise, int H);
int sins_fused_launch(const float* f0, const double* frame_phase, const float* c_amp, int64_t ctrl_stride, int H,
                      double sampling_rate, int round_fp32, const float* ir_allpass, int taps_allpass, float* harmonic,
                      const float* noise_in, const float* ir_noise, int taps_noise, float* noise_out, float* signal,
                      uint64_t seed, int64_t utt_off, int B, int nF, int P, cudaStream_t st);

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

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
    cudaEvent_t fork = nullptr, ir_done = nullptr, join = nullptr, join2 = nullptr;
    bool ok = false;
};
struct SideLanes {
    SideLane lane[64];
    ~SideLanes() {
        for (SideLane& l : lane) {
            if (l.fork) cudaEventDestroy(l.fork);
            if (l.ir_done) cudaEventDestroy(l.ir_done);
            if (l.join) cudaEventDestroy(l.join);
            if (l.join2) cudaEventDestroy(l.join2);
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
        good = good && cudaEventCreateWithFlags(&l.fork, cudaEventDisableTiming) == cudaSuccess;
        good = good && cudaEventCreateWithFlags(&l.ir_done, cudaEventDisableTiming) == cudaSuccess;
        good = good && cudaEventCreateWithFlags(&l.join, cudaEventDisableTiming) == cudaSuccess;
        good = good && cudaEventCreateWithFlags(&l.join2, cudaEventDisableTiming) == cudaSuccess;
        if (!good) { cudaGetLastError(); if (!l.hi) l.hi = (cudaStream_t)1; return nullptr; }
        l.ok = true;
    }
    return &l;
}
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
// workspace: sinusoids [B,T] | ir_allpass [B,nF,2(Ma-1)] | ir_noise [B,nF,2(Mn-1)]
// ---------------------------------------------------------------------------------------
extern "C" size_t b2d_sins_workspace_bytes(int B, int n_frames, int block, int n_mag_allpass, int n_mag_noise) {
    if (B <= 0 || n_frames <= 0 || block <= 0 || n_mag_allpass < 2 || n_mag_noise < 2) return 0;
    const size_t BT = (size_t)B * n_frames * block, BF = (size_t)B * n_frames;
    size_t n = b2d::align_up(BT * 4, 256) + b2d::align_up(BF * 2 * (n_mag_allpass - 1) * 4, 256) +
               b2d::align_up(BF * 2 * (n_mag_noise - 1) * 4, 256);
    // spectrum path (b2d_set_sins_impl(3) only): packed 1024-point spectra of both filters (512 float2 per frame)
    if (b2d::g_sins_impl.load(std::memory_order_relaxed) == 3 &&
        b2d::fir_spec_supported(block, 2 * (n_mag_allpass - 1), 2 * (n_mag_noise - 1)))
        n += 2 * b2d::align_up(b2d::fir_spec_floats(B, n_frames) * 4, 256);
    return n;
}

extern "C" int b2d_sins_synth(const float* f0_frames, const double* frame_phase, const float* c_amp,
                              const float* c_group_delay, const float* c_noise, int64_t ctrl_stride,
                              const float* noise_in, uint64_t seed, int64_t utterance_offset,
                              const float* dft_tables_allpass, const float* dft_tables_noise, int B, int n_frames,
                              int block, int n_harmonics, int n_mag_allpass, int n_mag_noise,
                              double sampling_rate, int round_fp32, float* signal, float* harmonic,
                              float* noise_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!workspace) return b2d::fail(B2D_ERR_NULL, "sins_synth: null workspace");
    const size_t need = b2d_sins_workspace_bytes(B, n_frames, block, n_mag_allpass, n_mag_noise);
    if (need == 0) return b2d::fail(B2D_ERR_SHAPE, "sins_synth: bad shape");
    if (workspace_bytes < need) return b2d::fail(B2D_ERR_WORKSPACE, "sins_synth: workspace %zu < %zu bytes", workspace_bytes, need);
    if ((reinterpret_cast<uintptr_t>(workspace) & 255u) != 0) return b2d::fail(B2D_ERR_ALIGN, "sins_synth: workspace must be 256-byte aligned");
    const size_t BT = (size_t)B * n_frames * block, BF = (size_t)B * n_frames;
    const int La = 2 * (n_mag_allpass - 1), Ln = 2 * (n_mag_noise - 1);
    char* ws = static_cast<char*>(workspace);
    float* sinus = reinterpret_cast<float*>(ws);
    float* ir_ap = reinterpret_cast<float*>(ws + b2d::align_up(BT * 4, 256));
    float* ir_n = reinterpret_cast<float*>(ws + b2d::align_up(BT * 4, 256) + b2d::align_up(BF * La * 4, 256));

    if (block % 256 != 0)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_synth: block size %d must be a multiple of 256", block);
    if (La != Ln && !noise_out) return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_synth: noise_out required when n_mag_allpass != n_mag_noise");
    cudaStream_t st = (cudaStream_t)stream;
    const int mode = b2d::g_overlap.load(std::memory_order_relaxed);
    b2d::SideLane* lane = mode != 0 ? b2d::side_lane() : nullptr;
    int nsplit = (mode < 0 ? -mode : mode);
    if (nsplit < 2 || !lane) nsplit = 1;
    if (nsplit > B) nsplit = B;
    cudaStream_t side = lane ? ((mode == 1 || mode < 0) ? lane->hi : lane->lo) : st;

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
    {
        const int simpl0 = b2d::g_sins_impl.load(std::memory_order_relaxed);
        const bool can_spec = b2d::fir_spec_supported(block, La, Ln) && b2d::fir_fft_selected();
        if (simpl0 == 3 && !can_spec)
            return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_synth: spectrum path needs block 512, <= 512 taps and the FFT-domain FIR");
        if (can_spec && simpl0 == 3) {
            const size_t spec_bytes = b2d::align_up(b2d::fir_spec_floats(B, n_frames) * 4, 256);
            float* spec_ap = reinterpret_cast<float*>(ws + b2d::align_up(BT * 4, 256) + b2d::align_up(BF * La * 4, 256) +
                                                      b2d::align_up(BF * Ln * 4, 256));
            float* spec_n = reinterpret_cast<float*>(reinterpret_cast<char*>(spec_ap) + spec_bytes);
            cudaStream_t q = lane ? lane->hi : st;
            cudaError_t fe = cudaSuccess;
            if (lane) {
                fe = cudaEventRecord(lane->fork, st);
                if (fe == cudaSuccess) fe = cudaStreamWaitEvent(q, lane->fork, 0);
                if (fe != cudaSuccess) return b2d::fail((int)fe, "sins_synth: fork: %s", cudaGetErrorString(fe));
            }
            int rc = irs(q, q);
            if (!rc) rc = b2d::ir_spectrum_launch(ir_ap, La, spec_ap, ir_n, Ln, spec_n, B, n_frames, q);
            if (lane) fe = cudaEventRecord(lane->join, q);
            int rcb = 0;
            if (!rc) rcb = bank(0, B, st);
            if (lane && fe == cudaSuccess) fe = cudaStreamWaitEvent(st, lane->join, 0);   // always join
            if (rc) return rc;
            if (rcb) return rcb;
            if (fe != cudaSuccess) return b2d::fail((int)fe, "sins_synth: join: %s", cudaGetErrorString(fe));
            return b2d::ltv_fir_fft_spec_launch(sinus, spec_ap, La, harmonic, noise_in, spec_n, Ln, noise_out, signal, seed,
                                                utterance_offset, B, n_frames, block, st);
        }
    }
    // ---- fused path: impulse responses (side by side on the two side streams), then ONE kernel: bank + both FIRs + mix ----
    const int simpl = b2d::g_sins_impl.load(std::memory_order_relaxed);
    const bool can_fuse = b2d::sins_fused_supported(block, La, Ln, n_harmonics) && b2d::fir_fft_selected();
    if (simpl == 2 && !can_fuse)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_synth: fused kernel needs block 512, <= 512 taps, <= 128 harmonics and the FFT-domain FIR");
    if (can_fuse && simpl == 2) {
        cudaError_t fe = cudaSuccess;
        int rc;
        if (lane) {
            fe = cudaEventRecord(lane->fork, st);
            if (fe == cudaSuccess) fe = cudaStreamWaitEvent(lane->hi, lane->fork, 0);
            if (fe == cudaSuccess) fe = cudaStreamWaitEvent(lane->lo, lane->fork, 0);
            if (fe != cudaSuccess) return b2d::fail((int)fe, "sins_synth: fork: %s", cudaGetErrorString(fe));
            rc = irs(lane->hi, lane->lo);
            fe = cudaEventRecord(lane->join, lane->hi);
            if (fe == cudaSuccess) fe = cudaStreamWaitEvent(st, lane->join, 0);
            if (fe == cudaSuccess) fe = cudaEventRecord(lane->join2, lane->lo);
            if (fe == cudaSuccess) fe = cudaStreamWaitEvent(st, lane->join2, 0);
        } else {
            rc = irs(st, st);
        }
        if (rc) return rc;
        if (fe != cudaSuccess) return b2d::fail((int)fe, "sins_synth: join: %s", cudaGetErrorString(fe));
        return b2d::sins_fused_launch(f0_frames, frame_phase, c_amp, ctrl_stride, n_harmonics, sampling_rate, round_fp32,
                                      ir_ap, La, harmonic, noise_in, ir_n, Ln, noise_out, signal, seed, utterance_offset,
                                      B, n_frames, block, st);
    }
    if (!lane) {                                       // in order on the caller's stream
        int rc = irs(st, st);
        if (!rc) rc = bank(0, B, st);
        if (!rc) rc = firs(0, B, st);
        return rc;
    }
    // fork: the side stream starts with the impulse responses of the whole batch (launched first: one 512-thread CTA per
    // SM, latency bound), the caller's stream with the first bank
    cudaError_t e = cudaEventRecord(lane->fork, st);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(side, lane->fork, 0);
    if (e != cudaSuccess) return b2d::fail((int)e, "sins_synth: fork: %s", cudaGetErrorString(e));
    // a small launch (one utterance, one pipeline chunk) leaves most SMs idle: its two impulse-response builds are latency
    // bound single waves, so they run side by side on the two side streams instead of one after the other
    const bool two_lanes = nsplit == 1 && (long long)B * n_frames <= (long long)b2d::num_sms() * 64;
    cudaStream_t side2 = two_lanes ? (side == lane->hi ? lane->lo : lane->hi) : side;
    if (two_lanes) {
        e = cudaStreamWaitEvent(side2, lane->fork, 0);
        if (e != cudaSuccess) return b2d::fail((int)e, "sins_synth: fork: %s", cudaGetErrorString(e));
    }
    int rc = irs(side, side2);
    cudaError_t je2 = cudaSuccess;
    if (two_lanes) {                                   // fold the second side stream into the first before its event
        je2 = cudaEventRecord(lane->join2, side2);
        if (je2 == cudaSuccess) je2 = cudaStreamWaitEvent(side, lane->join2, 0);
    }
    e = cudaEventRecord(lane->ir_done, side);
    if (e == cudaSuccess) e = je2;
    bool main_waited = false;
    for (int s = 0; s < nsplit && !rc && e == cudaSuccess; ++s) {
        const int b0 = (int)((long long)B * s / nsplit), b1 = (int)((long long)B * (s + 1) / nsplit);
        const bool on_side = (s & 1) != 0;
        cudaStream_t q = on_side ? side : st;
        rc = bank(b0, b1 - b0, q);
        if (!on_side && !main_waited) { e = cudaStreamWaitEvent(st, lane->ir_done, 0); main_waited = true; }
        if (!rc && e == cudaSuccess) rc = firs(b0, b1 - b0, q);
    }
    // always join, also after a failed launch: the caller's stream must not lose track of the side stream
    cudaError_t je = cudaEventRecord(lane->join, side);
    if (je == cudaSuccess) je = cudaStreamWaitEvent(st, lane->join, 0);
    if (rc) return rc;
    if (e != cudaSuccess) return b2d::fail((int)e, "sins_synth: event: %s", cudaGetErrorString(e));
    if (je != cudaSuccess) return b2d::fail((int)je, "sins_synth: join: %s", cudaGetErrorString(je));
    return 0;
}

// ---------------------------------------------------------------------------------------
// CombSub (old): comb source -> all-pass FIR -> dynamic-window harmonic FIR, + noise FIR
// (ddsp/vocoder.py:834-862).
// workspace: comb [B,T] | allpassed [B,T] | noise [B,T] | ir_ap | ir_h | ir_n
// ---------------------------------------------------------------------------------------
extern "C" int b2d_comb_source(const float*, const double*, int, int, int, double, int, float*, void*);

extern "C" size_t b2d_combsub_workspace_bytes(int B, int n_frames, int block, int n_mag_allpass,
                                              int n_mag_harmonic, int n_mag_noise) {
    if (B <= 0 || n_frames <= 0 || block <= 0 || n_mag_allpass < 2 || n_mag_harmonic < 2 || n_mag_noise < 2) return 0;
    const size_t BT = (size_t)B * n_frames * block, BF = (size_t)B * n_frames;
    return 3 * b2d::align_up(BT * 4, 256) + b2d::align_up(BF * 2 * (n_mag_allpass - 1) * 4, 256) +
           b2d::align_up(BF * 2 * (n_mag_harmonic - 1) * 4, 256) + b2d::align_up(BF * 2 * (n_mag_noise - 1) * 4, 256);
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
    const size_t need = b2d_combsub_workspace_bytes(B, n_frames, block, n_mag_allpass, n_mag_harmonic, n_mag_noise);
    if (need == 0) return b2d::fail(B2D_ERR_SHAPE, "combsub_synth: bad shape");
    if (workspace_bytes < need) return b2d::fail(B2D_ERR_WORKSPACE, "combsub_synth: workspace %zu < %zu bytes", workspace_bytes, need);
    if ((reinterpret_cast<uintptr_t>(workspace) & 255u) != 0) return b2d::fail(B2D_ERR_ALIGN, "combsub_synth: workspace must be 256-byte aligned");
    if (block % 256 != 0) return b2d::fail(B2D_ERR_UNSUPPORTED, "combsub_synth: block size %d must be a multiple of 256", block);
    const size_t BT = (size_t)B * n_frames * block, BF = (size_t)B * n_frames;
    const int La = 2 * (n_mag_allpass - 1), Lh = 2 * (n_mag_harmonic - 1), Ln = 2 * (n_mag_noise - 1);
    char* ws = static_cast<char*>(workspace);
    const size_t sBT = b2d::align_up(BT * 4, 256);
    float* comb = reinterpret_cast<float*>(ws);
    float* allp = reinterpret_cast<float*>(ws + sBT);
    float* nbuf = noise_out ? noise_out : reinterpret_cast<float*>(ws + 2 * sBT);
    float* ir_ap = reinterpret_cast<float*>(ws + 3 * sBT);
    float* ir_h = reinterpret_cast<float*>(ws + 3 * sBT + b2d::align_up(BF * La * 4, 256));
    float* ir_n = reinterpret_cast<float*>(ws + 3 * sBT + b2d::align_up(BF * La * 4, 256) + b2d::align_up(BF * Lh * 4, 256));
    cudaStream_t st = (cudaStream_t)stream;

    // the dynamic-window impulse response (the largest of the three builds) is only needed by the LAST filter: it runs on
    // the internal side stream beside the all-pass / noise stage and is joined right before the harmonic filter
    b2d::SideLane* lane = b2d::g_overlap.load(std::memory_order_relaxed) != 0 ? b2d::side_lane() : nullptr;
    cudaError_t je = cudaSuccess;
    if (lane) {
        je = cudaEventRecord(lane->fork, st);
        if (je == cudaSuccess) je = cudaStreamWaitEvent(lane->hi, lane->fork, 0);
        if (je != cudaSuccess) return b2d::fail((int)je, "combsub_synth: fork: %s", cudaGetErrorString(je));
    }
    const int rch = b2d_ir_build(c_harmonic, ctrl_stride, B2D_IR_MAG_DYNAMIC, f0_frames, dft_tables_harmonic, B, n_frames,
                                 n_mag_harmonic, sampling_rate, ir_h, lane ? (void*)lane->hi : stream);
    if (lane) je = cudaEventRecord(lane->join, lane->hi);
    // from here on every return path must first join the side stream
    auto joined = [&](int code) -> int {
        if (lane && je == cudaSuccess) je = cudaStreamWaitEvent(st, lane->join, 0);
        if (code) return code;
        if (rch) return rch;
        if (je != cudaSuccess) return b2d::fail((int)je, "combsub_synth: join: %s", cudaGetErrorString(je));
        return 0;
    };
    int rc = b2d_comb_source(f0_frames, frame_phase, B, n_frames, block, sampling_rate, round_fp32, comb, stream);
    if (rc) return joined(rc);
    rc = b2d_ir_build(c_group_delay, ctrl_stride, B2D_IR_ALLPASS, nullptr, dft_tables_allpass, B, n_frames,
                      n_mag_allpass, sampling_rate, ir_ap, stream);
    if (rc) return joined(rc);
    rc = b2d_ir_build(c_noise, ctrl_stride, B2D_IR_MAG_HANN, nullptr, dft_tables_noise, B, n_frames, n_mag_noise,
                      sampling_rate, ir_n, stream);
    if (rc) return joined(rc);
    // all-pass on the comb and the noise filter: one launch when the tap counts agree
    if (La == Ln) {
        rc = b2d::ltv_fir_launch(comb, ir_ap, La, allp, noise_in, ir_n, Ln, nbuf, nullptr, nullptr, seed,
                                 utterance_offset, B, n_frames, block, st);
        if (rc) return joined(rc);
    } else {
        rc = b2d::ltv_fir_launch(comb, ir_ap, La, allp, nullptr, nullptr, 0, nullptr, nullptr, nullptr, seed,
                                 utterance_offset, B, n_frames, block, st);
        if (rc) return joined(rc);
        rc = b2d::ltv_fir_launch(noise_in, ir_n, Ln, nbuf, nullptr, nullptr, 0, nullptr, nullptr, nullptr, seed,
                                 utterance_offset, B, n_frames, block, st);
        if (rc) return joined(rc);
    }
    rc = joined(0);
    if (rc) return rc;
    // harmonic magnitude filter on the all-passed comb; signal = harmonic + noise
    return b2d::ltv_fir_launch(allp, ir_h, Lh, harmonic, nullptr, nullptr, 0, nullptr, nbuf, signal, seed,
                               utterance_offset, B, n_frames, block, st);
}
