/*
 * b200ddsp.h -- C ABI of libb200ddsp.so: the H100 (sm_90a) DDSP harmonic-plus-noise
 * synthesis kernels behind the reference's Sins / CombSub / CombSubSuperFast / SineGen
 * forward() calls (yxlllc/DDSP-SVC).
 *
 * The reference has no FFI of its own: its "operator API" for this path is the Python
 * module call (ddsp/vocoder.py:556,653,811; nsf_hifigan/models.py:150).  This header is
 * what a maintainer binds (ctypes, see INTEGRATION.md) to replace the tensor code inside
 * those forward() methods.  Each entry point cites the reference lines it replaces.
 *
 * Conventions
 *  - plain C types only; every pointer is a DEVICE pointer to contiguous fp32 data unless
 *    stated otherwise; `stream` is a cudaStream_t passed as void*.
 *  - the library never allocates or frees device memory and never synchronises the stream.
 *    Its entry points are re-entrant from any host thread (the reference is called from the
 *    audio-callback thread of gui.py:376-414 and from Flask): the last-error string is
 *    thread-local, and the only process-wide state is (i) a mutex-protected, per-device
 *    cache of internal fork/join streams and events (b2d_sins_synth runs independent
 *    kernels side by side and joins them on the caller's stream before returning) and
 *    (ii) the b2d_set_* implementation selectors: atomics, each read ONCE at the top of a
 *    call.  The selectors exist for A/B measurements and tests; every setting computes the
 *    same function, so flipping one from another thread changes which kernel a later call
 *    uses, never a result.
 *  - return value: 0 = ok, <0 = argument error (B2D_ERR_*), >0 = cudaError_t of the failed
 *    launch.  No exceptions or aborts cross the ABI.  b2d_last_error() describes the last
 *    failure on the calling thread.
 *  - "ctrl_stride": raw control tensors arrive as strided views of ONE dense
 *    [B, n_frames, n_out] tensor (torch.split in ddsp/unit2control.py:12-23); every control
 *    pointer therefore comes with the element stride between consecutive frames.
 *  - T = n_frames * block.  Utterances (batch rows) are independent.
 */
#ifndef B200DDSP_H
#define B200DDSP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2D_VERSION 100

#define B2D_ERR_NULL        (-1)  /* required pointer is NULL                         */
#define B2D_ERR_SHAPE       (-2)  /* non-positive or inconsistent dimension           */
#define B2D_ERR_ALIGN       (-3)  /* pointer / stride not aligned as required         */
#define B2D_ERR_UNSUPPORTED (-4)  /* configuration outside what the kernels implement */
#define B2D_ERR_WORKSPACE   (-5)  /* workspace too small                              */

/* impulse-response construction modes (b2d_ir_build) */
#define B2D_IR_ALLPASS      0  /* H = exp(j*cumsum(pi*tanh(c))), no window   (ddsp/vocoder.py:581,599) */
#define B2D_IR_MAG_HANN     1  /* H = exp(c)/128, periodic Hann window        (ddsp/vocoder.py:582,606) */
#define B2D_IR_MAG_DYNAMIC  2  /* H = exp(c), per-frame raised-cosine window  (ddsp/vocoder.py:835,849-851) */

int         b2d_version(void);
const char* b2d_last_error(void);

/* ---------------------------------------------------------------------------------------
 * Exciter phase at frame rate.                       replaces ddsp/vocoder.py:564-575
 * (same code at :743-753 and :819-829).
 *   frame_phase[b,k] = sum_{i<k} (P f_i + (f_{i+1}-f_i)(P-1)/2)/sr  (+ initial_phase/2pi),
 *                      unwrapped cycles, fp64  -- the closed form of the reference's
 *                      per-sample fp64 cumsum of the linearly upsampled f0.
 *   phase_frames[b,k] = 2*pi*fp32(wrap(x[k*P]))  -- the tensor handed to Unit2Control.
 * f0_frames [B, n_frames] Hz.  initial_phase: NULL or [B] radians.
 * round_fp32: 0 = infer=True (fp64 phase), 1 = infer=False (phase rounded to fp32 before
 * wrapping, ddsp/vocoder.py:568).
 */
int b2d_phase_scan(const float* f0_frames, const float* initial_phase, int B, int n_frames,
                   int block, double sampling_rate, int round_fp32,
                   double* frame_phase, float* phase_frames, void* stream);

/* ---------------------------------------------------------------------------------------
 * Additive sinusoid bank.                            replaces ddsp/vocoder.py:580,585-594
 * and ddsp/core.py:66-77 (upsample, remove_above_fmax).
 *   sinusoids[b,t] = sum_{h=1..H} sin(h * phase[t]) * up(A)[t,h],
 *   A[k,h] = exp(c_amp[k,h])/128 * (1[f0[k]*h < sr/2] + 1e-7).
 * c_amp: raw 'amplitudes' control, [B, n_frames, H] with frame stride ctrl_stride.
 */
int b2d_sins_bank(const float* f0_frames, const double* frame_phase, const float* c_amp,
                  int64_t ctrl_stride, int B, int n_frames, int block, int n_harmonics,
                  double sampling_rate, int round_fp32, float* sinusoids, void* stream);

/* ---------------------------------------------------------------------------------------
 * Frame-wise impulse responses from raw controls.    replaces ddsp/core.py:254-270
 * (frequency_impulse_response) + :185-237 / :240-251 (windows) and the activations at
 * ddsp/vocoder.py:581-582,599,606,835-836,845,849-851.
 *   ir[b,k,:] has L = 2*(n_mag-1) taps in causal form.
 * dft_tables: device buffer of b2d_dft_tables_bytes(n_mag) bytes filled once by
 * b2d_dft_tables() (constant cos/sin matrices of the L-point inverse real DFT).
 * f0_frames is only read in mode B2D_IR_MAG_DYNAMIC (window half-width 1.5*sr/(f0+1e-3)).
 */
/* Two implementations: wgmma tensor cores (3xTF32; default when the accumulators fit the registers)
 * and CUDA cores.  b2d_set_ir_impl: 0 = automatic, 1 = CUDA cores, 2 = tensor cores (test knob).
 * The table buffer (256-byte aligned) holds the constant matrices for both. */
int    b2d_set_ir_impl(int impl);
size_t b2d_dft_tables_bytes(int n_mag);
int    b2d_dft_tables(int n_mag, float* dft_tables, void* stream);
int    b2d_ir_build(const float* c, int64_t ctrl_stride, int mode, const float* f0_frames,
                    const float* dft_tables, int B, int n_frames, int n_mag,
                    double sampling_rate, float* ir, void* stream);

/* ---------------------------------------------------------------------------------------
 * Linear time-varying FIR (frequency_filter's convolution).   replaces ddsp/core.py:120-182
 * (fft_convolve: Bartlett-windowed 50%-overlap frames, per-frame IR, overlap-add, crop
 * with delay L/2).  The linear convolution it defines is
 *   y[n] = sum_tau ((1-phi_m) h_f[tau] + phi_m h_{f+1}[tau]) x[m],  m = n + L/2 - tau,
 *   f = floor(m/P), phi_m = (m mod P)/P, h_{nF} := h_{nF-1}, x = 0 outside [0,T).
 * Up to two independent filters ("jobs") run in one launch and their outputs can be
 * summed into `mix` (signal = harmonic + noise, ddsp/vocoder.py:609).
 * x1 / x2: input [B, T]; NULL means "white noise U(-1,1) generated in-kernel" from
 * Philox4x32-10 keyed by (seed, utterance index + utterance_offset, sample index)
 * (replaces torch.rand_like(...)*2-1, ddsp/vocoder.py:603).
 * y1 / y2 / mix may be NULL when that output is not wanted; job 2 is skipped when ir2 is
 * NULL.
 */
int b2d_ltv_fir(const float* x1, const float* ir1, int taps1, float* y1,
                const float* x2, const float* ir2, int taps2, float* y2,
                float* mix, uint64_t seed, int64_t utterance_offset,
                int B, int n_frames, int block, void* stream);

/* Kernel selection for b2d_ltv_fir and the synthesizer drivers.  0 = automatic: the FFT-domain kernel
 * (ltv_fir_fft.cu: per input hop one N-point FFT per signal, the impulse responses' spectra and one inverse FFT per
 * pair of hops; N = 1024 up to 512 taps, 2048 up to 1024 taps; ~4x fewer instructions than the direct form)
 * when the block size is 512 and no filter has more than
 * 1024 taps, otherwise the CUDA-core direct form (block size multiple of 256).  1 = CUDA-core direct form
 * (16 outputs per thread, register-pair FMAs), 2 = wgmma tensor cores (3xTF32, block size 512; correct but
 * operand-bandwidth bound and ~3x slower, see DESIGN.md), 3 = the older 8-outputs-per-thread scalar-FFMA direct form,
 * 4 = FFT-domain kernel wherever it applies.  B2D_FIR_AUTO=cuda in the environment makes 0 mean 1.
 * Process-wide test/diagnostic knob. */
int b2d_set_fir_impl(int impl);

/* Same result by the plain one-thread-per-sample formula (any block size / tap count);
 * used as the fallback for configurations the tiled kernel does not cover and as an
 * on-device cross-check. One job only. */
int b2d_ltv_fir_generic(const float* x, const float* ir, int taps, float* y,
                        int B, int n_frames, int block, void* stream);

/* ---------------------------------------------------------------------------------------
 * Whole Sins synthesizer after Unit2Control.         replaces ddsp/vocoder.py:580-611
 * Raw controls in, three waveforms out (any of signal/harmonic/noise_out may be NULL).
 * noise_in: [B, T] uniform(-1,1) samples (parity mode) or NULL (in-kernel Philox).
 * workspace: b2d_sins_workspace_bytes(...) bytes, 256-byte aligned.
 */
size_t b2d_sins_workspace_bytes(int B, int n_frames, int block, int n_mag_allpass, int n_mag_noise);
int    b2d_sins_synth(const float* f0_frames, const double* frame_phase,
                      const float* c_amp, const float* c_group_delay, const float* c_noise,
                      int64_t ctrl_stride, const float* noise_in, uint64_t seed,
                      int64_t utterance_offset, const float* dft_tables_allpass,
                      const float* dft_tables_noise, int B, int n_frames, int block,
                      int n_harmonics, int n_mag_allpass, int n_mag_noise,
                      double sampling_rate, int round_fp32,
                      float* signal, float* harmonic, float* noise_out,
                      void* workspace, size_t workspace_bytes, void* stream);

/* Backward of b2d_sins_synth in the training phase (round_fp32 = 1, infer=False) with respect to
 * the three raw controls.                            ddsp/vocoder.py:580-611 under autograd
 * grad_ctrl: dense [B, n_frames, H + Ma + Mn] = amplitudes | group_delay | noise_magnitude (the
 * split_to_dict layout), every element written.  grad_signal / grad_harmonic / grad_noise: [B, T]
 * cotangents of the three outputs, NULL = zero.  forward_workspace: what b2d_sins_synth filled
 * for the same arguments (its impulse responses, and its sinusoids unless
 * forward_has_sinusoids = 0: the fused variant, b2d_set_sins_impl(2), does not store them and the
 * bank is rerun into `workspace`).  f0_frames, frame_phase, controls, noise_in, seed and
 * utterance_offset: those of the forward call (the in-kernel noise is regenerated).  Built for
 * block 512, 2 <= n_mag <= 257, H <= 512.  Deterministic: no atomics; the result depends neither
 * on the grid nor on b2d_set_overlap / b2d_set_sins_impl. */
size_t b2d_sins_synth_backward_workspace_bytes(int B, int n_frames, int block);
int    b2d_sins_synth_backward(const float* f0_frames, const double* frame_phase, const float* c_amp,
                               const float* c_group_delay, const float* c_noise, int64_t ctrl_stride,
                               const float* noise_in, uint64_t seed, int64_t utterance_offset,
                               const void* forward_workspace, int forward_has_sinusoids,
                               const float* grad_signal, const float* grad_harmonic,
                               const float* grad_noise, int B, int n_frames, int block,
                               int n_harmonics, int n_mag_allpass, int n_mag_noise,
                               double sampling_rate, float* grad_ctrl, void* workspace,
                               size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * NSF-HiFiGAN SineGen f0 excitation.                replaces nsf_hifigan/models.py:134-165
 * (SineGen._f02sine + forward).  f0 [B, n_frames] (Hz, 0 = unvoiced), piecewise constant per
 * frame of `upp` samples; out [B, n_frames*upp, dim], dim = harmonic_num + 1 <= 16.
 * rand_ini [dim]: the random initial phases in cycles (element 0 = 0), drawn by the caller
 * (reference: torch.rand(1,1,dim), models.py:144-145).
 * noise_in [B, T, dim]: N(0,1) samples (parity mode) or NULL = in-kernel Philox + Box-Muller
 * (replaces torch.randn_like, models.py:163).
 * acc_workspace: B*n_frames floats (per-frame wrapped phase advance, models.py:139-141).
 */
int b2d_sinegen(const float* f0, const float* rand_ini, const float* noise_in, uint64_t seed,
                int64_t utterance_offset, int B, int n_frames, int upp, int dim,
                double sampling_rate, float sine_amp, float noise_std, float voiced_threshold,
                float* acc_workspace, float* out, void* stream);

/* ---------------------------------------------------------------------------------------
 * CombSub (old version): comb-tooth source.          replaces ddsp/vocoder.py:819-829,839-840
 *   comb[b,t] = sinc(sr * x[t] / (f0_up[t] + 1e-3)), x = wrapped phase (cycles, fp32).
 */
int b2d_comb_source(const float* f0_frames, const double* frame_phase, int B, int n_frames,
                    int block, double sampling_rate, int round_fp32, float* comb, void* stream);

/* Whole old-CombSub synthesizer after Unit2Control.  replaces ddsp/vocoder.py:834-862
 * comb -> all-pass (group delay) -> harmonic magnitude filter with the per-frame dynamic
 * window (half width 1.5*sr/(f0+1e-3)); noise -> Hann-windowed noise filter; signal = sum.
 * signal/harmonic/noise_out may be NULL.  workspace: b2d_combsub_workspace_bytes bytes.
 */
size_t b2d_combsub_workspace_bytes(int B, int n_frames, int block, int n_mag_allpass,
                                   int n_mag_harmonic, int n_mag_noise);
int    b2d_combsub_synth(const float* f0_frames, const double* frame_phase,
                         const float* c_group_delay, const float* c_harmonic, const float* c_noise,
                         int64_t ctrl_stride, const float* noise_in, uint64_t seed,
                         int64_t utterance_offset, const float* dft_tables_allpass,
                         const float* dft_tables_harmonic, const float* dft_tables_noise,
                         int B, int n_frames, int block, int n_mag_allpass, int n_mag_harmonic,
                         int n_mag_noise, double sampling_rate, int round_fp32,
                         float* signal, float* harmonic, float* noise_out,
                         void* workspace, size_t workspace_bytes, void* stream);

/* Backward of b2d_combsub_synth in the training phase (round_fp32 = 1, infer=False) with respect
 * to the three raw controls.                         ddsp/vocoder.py:834-862 under autograd
 * grad_ctrl: dense [B, n_frames, Ma + Mh + Mn] = group_delay | harmonic_magnitude |
 * noise_magnitude (the split_to_dict layout), every element written.  grad_signal /
 * grad_harmonic / grad_noise: [B, T] cotangents of the three outputs, NULL = zero.
 * forward_workspace: what b2d_combsub_synth filled for the same arguments (its comb, all-passed
 * comb and impulse responses).  f0_frames, controls, noise_in, seed and utterance_offset: those of
 * the forward call (the in-kernel noise is regenerated).  workspace: dL/d(all-passed comb), [B, T].
 * Built for block 512, 2 <= n_mag <= 513 (up to 1024 taps).  Deterministic: no atomics; the
 * result depends neither on the grid nor on b2d_set_overlap. */
size_t b2d_combsub_synth_backward_workspace_bytes(int B, int n_frames, int block);
int    b2d_combsub_synth_backward(const float* f0_frames, const float* c_group_delay,
                                  const float* c_harmonic, const float* c_noise, int64_t ctrl_stride,
                                  const float* noise_in, uint64_t seed, int64_t utterance_offset,
                                  const void* forward_workspace, const float* grad_signal,
                                  const float* grad_harmonic, const float* grad_noise, int B,
                                  int n_frames, int block, int n_mag_allpass, int n_mag_harmonic,
                                  int n_mag_noise, double sampling_rate, float* grad_ctrl,
                                  void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * CombSubSuperFast (what configs/combsub.yaml selects).   replaces ddsp/vocoder.py:639-710
 * Two steps around Unit2Control, like the reference:
 *  b2d_superfast_scan : per-frame source parameters (s, ds, wrapped phase advance) into
 *                       `workspace` (b2d_superfast_workspace_bytes) and phase_frames [B,nF]
 *                       = 2*pi*rad[:, :, 0]                      (fast_source_gen, :639-651)
 *  b2d_superfast_synth: comb source -> STFT (2048/512, Hann, reflect) of comb and of N(0,1)
 *                       noise -> Y = X exp(m_h + j pi p_h) + N exp(m_n + j pi p_n)/128 (last
 *                       frame repeated) -> iSTFT -> signal [B, n_frames*block]   (:666-708)
 * The four raw controls [B, n_frames, win_length/2+1] share ctrl_stride.
 * noise_in [B,T] N(0,1) (parity) or NULL (in-kernel Philox + Box-Muller).
 * Only win_length = 2048, block = 512 is implemented (B2D_ERR_UNSUPPORTED otherwise).
 */
size_t b2d_superfast_workspace_bytes(int B, int n_frames);
int    b2d_superfast_scan(const float* f0_frames, int B, int n_frames, int block,
                          double sampling_rate, void* workspace, float* phase_frames, void* stream);
int    b2d_superfast_synth(const void* workspace, const float* c_harmonic_magnitude,
                           const float* c_harmonic_phase, const float* c_noise_magnitude,
                           const float* c_noise_phase, int64_t ctrl_stride, const float* noise_in,
                           uint64_t seed, int64_t utterance_offset, int B, int n_frames, int block,
                           int win_length, float* signal, void* stream);
/* Backward of b2d_superfast_synth with respect to the four raw controls (training; no gradient with respect to
 * f0).  Same workspace, controls, noise_in / seed / utterance_offset as the forward call (the comb and noise
 * spectra are recomputed, the in-kernel noise stream is regenerated); grad_signal = dL/dsignal [B, T] (T =
 * n_frames*block).  grad_ctrl [B, n_frames, 4*(win_length/2+1)] receives dL/d(harmonic_magnitude |
 * harmonic_phase | noise_magnitude | noise_phase) per frame; it is overwritten, deterministically (no atomics).
 * grad_signal, grad_ctrl, noise_in and workspace must be 16-byte aligned. */
int    b2d_superfast_synth_backward(const void* workspace, const float* c_hm, const float* c_hp,
                                    const float* c_nm, const float* c_np, int64_t ctrl_stride,
                                    const float* noise_in, uint64_t seed, int64_t utterance_offset,
                                    const float* grad_signal, int B, int n_frames, int block, int win_length,
                                    float* grad_ctrl, void* stream);

/* SineGen fused with the tail of SourceModuleHnNSF.   replaces nsf_hifigan/models.py:201-204
 * (sine_merge = tanh(l_linear(sine_wavs))) on top of b2d_sinegen: merged [B, n_frames*upp] =
 * tanh(linear_bias + sum_h linear_weight[h] * sine_wavs[..., h]); the [B, T, dim] tensor is never
 * materialised (4 instead of 36 bytes per sample).  SURVEY 8(f) rank 2 ("next") fusion. */
int b2d_source_module(const float* f0, const float* rand_ini, const float* noise_in, uint64_t seed,
                      int64_t utterance_offset, int B, int n_frames, int upp, int dim,
                      double sampling_rate, float sine_amp, float noise_std, float voiced_threshold,
                      const float* linear_weight, float linear_bias, float* acc_workspace,
                      float* merged, void* stream);

/* CombSubFast STFT-domain filter.   replaces ddsp/vocoder.py:758-784
 * comb [B, T] is the comb-tooth source of b2d_comb_source (the same expression as :764 on the same phase,
 * :743-751 = b2d_phase_scan); controls are raw Unit2Control outputs [B, n_frames, block+1] with a common frame
 * stride; noise_in [B, T] uniform(-1,1) or NULL = in-kernel Philox (same stream as b2d_ltv_fir).
 * Frames of 2*block at hop block, sqrt-Hann analysis and synthesis windows, filter row min(q, n_frames-1),
 * overlap-add cropped by block on both sides.  block must be 512. */
int b2d_combsubfast_filter(const float* comb, const float* c_harmonic_magnitude, const float* c_harmonic_phase,
                           const float* c_noise_magnitude, int64_t ctrl_stride, const float* noise_in,
                           uint64_t seed, int64_t utterance_offset, int B, int n_frames, int block,
                           float* signal, void* stream);
/* Backward of b2d_combsubfast_filter with respect to the three raw controls (training; no gradient with respect to
 * comb).  Same comb, controls, noise_in / seed / utterance_offset as the forward call (the source spectra are
 * recomputed, the in-kernel noise stream is regenerated); grad_signal = dL/dsignal [B, T] (T = n_frames*block).
 * grad_ctrl [B, n_frames, 3*(block+1)] receives dL/d(harmonic_magnitude | harmonic_phase | noise_magnitude) per
 * frame; it is overwritten, deterministically (no atomics), bit-identically for any batch split.
 * comb, grad_signal, grad_ctrl and noise_in must be 16-byte aligned.  block must be 512. */
int b2d_combsubfast_filter_backward(const float* comb, const float* c_hm, const float* c_hp, const float* c_nm,
                                    int64_t ctrl_stride, const float* noise_in, uint64_t seed,
                                    int64_t utterance_offset, const float* grad_signal, int B, int n_frames,
                                    int block, float* grad_ctrl, void* stream);

/* Arithmetic of the shared-memory FFT kernels (ltv_fir_fft, superfast, combsubfast): 1 (default) = the
 * "packed" instantiations, 0 = the scalar ones; Hopper has no packed FP32 add, so both use scalar complex additions.  B2D_FFT_ARITH=scalar in the environment selects 0 as the initial value.  Process-wide test/diagnostic knob
 * (atomic, read once per call). */
int b2d_set_fft_arith(int packed);

/* ---- caller-side prologue / epilogue (SURVEY 8f rank 2) -------------------------------------------------------------
 * Volume_Extractor.extract (ddsp/vocoder.py:147-157): audio [B, n_samples] -> volume [B, n_samples / hop + 1],
 * volume[n] = sqrt(mean(pad_reflect(audio^2, hop/2, (hop+1)/2)[n hop : (n+1) hop])). */
int b2d_volume_extract(const float* audio, int B, int n_samples, int hop, float* volume, void* stream);

/* Silence mask at frame rate (main.py:211-213): mask[n] = max over frames n-4..n+4 (clamped) of (volume > threshold). */
int b2d_volume_mask(const float* volume, int B, int n_frames, float threshold, float* mask_frames, void* stream);

/* `seg_output *= upsample(mask, block)[frame_offset*block : (frame_offset+n_frames)*block]` in place (main.py:215,260;
 * upsample = ddsp/core.py:66-70: linear, last frame held).  signal [B, n_frames*block], mask_frames [B, n_mask_frames]. */
int b2d_mask_apply(float* signal, const float* mask_frames, int B, int n_mask_frames, int frame_offset, int n_frames,
                   int block, void* stream);

/* Segment cross-fade (main.py:142-149): out[0 : idx + len_b] = a[:idx] | (1-k) a[idx:] + k b[:len_a-idx] | b[len_a-idx:],
 * k = linspace(0, 1, len_a - idx) evaluated in fp64.  Requires 0 <= idx < len_a and len_a - idx <= len_b. */
int b2d_cross_fade(const float* a, int64_t len_a, const float* b, int64_t len_b, int64_t idx, float* out, void* stream);

/* ---- fused frame-rate kernels of the control network (Unit2Control inference, ddsp/unit2control.py:84-109 with
 * ddsp/pcmer.py / diffusion/model_conformer_naive.py): everything that is not a plain GEMM.  Activations are token-major
 * [B, T, C] fp32; the model width is 256 as in the reference.
 * u2c_embed (:93-102): x [B*T, 256] += f0_embed(log(1 + f0/700)) + phase_embed(phase/pi) + volume_embed(volume) + spk
 *   (+ aug_embed(aug_shift/5)); embed_table [7, 256] = f0 w, f0 b, phase w, phase b, volume w, volume b, aug w;
 *   spk [spk_rows, 256] (spk_rows 1 or B) or NULL; aug_shift [B] or NULL.
 * u2c_groupnorm_lrelu (:50-52): GroupNorm(groups, C = 256) with statistics over (C/groups channels x T) of each utterance,
 *   then LeakyReLU(slope), in place; stats_ws: B * groups * 2 doubles of scratch.
 * u2c_layernorm: LayerNorm over the last dimension C (multiple of 32, <= 1024) of n_tokens rows.
 * u2c_glu_dwconv_silu (pcmer.py:211-215): in [B, T, 2 Ci] -> GLU -> depthwise Conv1d(k = 31, zero padding 15/15,
 *   weight [Ci, 31], bias [Ci]) -> SiLU -> out [B, T, Ci]; Ci multiple of 128.
 * u2c_softmax_features (pcmer.py:13-48): performer softmax-kernel feature map, in place on projected = (d^-1/4 data) proj^T
 *   [rows, n_features] with data [rows, dim_head]: query rows ratio (exp(p - diag - rowmax) + eps), key rows
 *   ratio exp(p - diag + eps), diag = |data|^2 / (2 sqrt(d)), ratio = n_features^-1/2. */
/* x [n] -> hi, lo [n]: x = hi + lo up to 2^-22 |x| with both parts exactly representable in TF32 (round to nearest even);
 * the operand preparation of 3xTF32 GEMMs (hi hi + lo hi + hi lo on the tensor cores = fp32-grade products).
 * A NaN gives the TF32 quiet NaN in both parts, +-inf gives (+-inf, +0); finite values at or above (2 - 2^-11) 2^127
 * round to hi = +-inf, lo = -+inf. */
int b2d_split_tf32(const float* x, float* hi, float* lo, size_t n, void* stream);
int b2d_u2c_embed(float* x, const float* f0, const float* phase, const float* volume, const float* embed_table,
                  const float* spk, int spk_rows, const float* aug_shift, int B, int T, void* stream);
int b2d_u2c_groupnorm_lrelu(float* x, int B, int T, int C, int groups, const float* gamma, const float* beta, float eps,
                            float slope, double* stats_ws, void* stream);
int b2d_u2c_layernorm(const float* x, float* y, int n_tokens, int C, const float* gamma, const float* beta, float eps,
                      void* stream);
int b2d_u2c_glu_dwconv_silu(const float* in, const float* weight, const float* bias, float* out, int B, int T,
                            int inner_channels, int kernel_size, void* stream);
int b2d_u2c_softmax_features(float* projected, const float* data, int rows, int n_features, int dim_head, int is_query,
                             float eps, void* stream);
/* Fused non-causal linear attention of the performer layers (ddsp/pcmer.py:220-229), one CTA per (utterance, head):
 * q_features, k_features [B*H, T, n_features] (the feature maps above), v [B*H, T, dim_head] ->
 * out [B, T, H, dim_head] = (q' . (k'^T v)) / (q' . sum_t k' + eps).  dim_head must be 64, n_features <= 272. */
int b2d_u2c_linear_attention(const float* q_features, const float* k_features, const float* v, float* out, int B, int H,
                             int T, int n_features, int dim_head, float eps, void* stream);

/* ---- backward of the control network with the convolution-only decoder (unit2control_bwd.cu): the adjoints of the
 * kernels above that the naive decoder runs; the GEMM adjoints are library GEMMs of the caller.  No atomics: sums over
 * tokens are taken per fixed slab of tokens into the workspace, then added in slab order in fp64, so every result is
 * bit-identical from run to run and independent of the device.  `ws` is scratch of at least
 * b2d_u2c_backward_workspace_bytes(B, T, inner_channels, max_cols) bytes (enough for each call below with n_tokens = B T,
 * that inner_channels, and n_cols <= max_cols; 0 = bad shape); too small a workspace returns B2D_ERR_WORKSPACE.
 * u2c_glu_dwconv_silu_backward: h [B, T, 2 Ci] is the forward's INPUT (the stage is recomputed from it), gout [B, T, Ci]
 *   the cotangent of its output -> gh [B, T, 2 Ci] and dwb [Ci, 32]: 31 tap gradients, then the bias gradient.
 * u2c_colsum: out [n_cols] = column sums of g [n_tokens, n_cols] (the bias gradient of a GEMM).
 * u2c_layernorm_backward (C = 256): x the forward's input, gy the cotangent of its output -> gx, and dgamma_dbeta [2, C].
 * u2c_groupnorm_lrelu_backward (C = 256): x_pre [B, T, C] the activation BEFORE the in-place forward, stats the
 *   B * groups * 2 doubles the forward left in stats_ws, gy the cotangent of the LeakyReLU output -> gx, dgamma_dbeta [2, C].
 * u2c_embed_backward: gx [B*T, 256] the cotangent of u2c_embed's output (which is also the cotangent of its input x) ->
 *   dtable [7, 256], the gradient of embed_table, and rowsum [B, 256] = per-utterance sums of gx (the gradient of each
 *   utterance's speaker row); aug_shift [B] or NULL as in the forward.
 * u2c_conv3_fold: adjoint of gathering (x[t-1], x[t], x[t+1]) (zero padded) into rows of 3 * channels:
 *   gx[t] = gcat[t+1][0:I] + gcat[t][I:2I] + gcat[t-1][2I:3I]. */
size_t b2d_u2c_backward_workspace_bytes(int B, int T, int inner_channels, int max_cols);
int b2d_u2c_glu_dwconv_silu_backward(const float* h, const float* weight, const float* bias, const float* gout, float* gh,
                                     float* dwb, int B, int T, int inner_channels, int kernel_size, void* ws, size_t ws_bytes,
                                     void* stream);
int b2d_u2c_colsum(const float* g, int n_tokens, int n_cols, float* out, void* ws, size_t ws_bytes, void* stream);
int b2d_u2c_layernorm_backward(const float* x, const float* gy, const float* gamma, float eps, int n_tokens, int C, float* gx,
                               float* dgamma_dbeta, void* ws, size_t ws_bytes, void* stream);
int b2d_u2c_groupnorm_lrelu_backward(const float* x_pre, const double* stats, const float* gamma, const float* beta, float eps,
                                     float slope, const float* gy, int B, int T, int C, int groups, float* gx,
                                     float* dgamma_dbeta, void* ws, size_t ws_bytes, void* stream);
int b2d_u2c_embed_backward(const float* gx, const float* f0, const float* phase, const float* volume, const float* aug_shift,
                           int B, int T, float* dtable, float* rowsum, void* ws, size_t ws_bytes, void* stream);
int b2d_u2c_conv3_fold(const float* gcat, int B, int T, int channels, float* gx, void* stream);

/* ---- backward of the PCmer decoder's performer attention (pcmer_bwd.cu): the stages between the caller's library GEMMs.
 * Rows are (b, h, t) of B * H * T; dim_head must be 64.  No atomics and no workspace: one warp per row, so every result is
 * bit-identical from run to run.
 * u2c_attn_readout_backward: out = (phi_q ctx) d_inv with d_inv [B, H, T] = 1 / (phi_q . ksum + 1e-8); g_out and out
 *   [B, T, H, 64] token-major -> gn [B, H, T, 65]: g_out d_inv, then g_D = -(g_out . out) d_inv.
 * u2c_softmax_features_backward: adjoint of u2c_softmax_features.  g [rows, n_features] (n_features <= 288) holds the
 *   cotangent of the features on entry and that of `projected` on return; features the forward's output, data its input
 *   [rows, 64]; the full cotangent is g + scal[row] vec[row / T] (queries: scal = g_D, vec = ksum [rows / T, n_features])
 *   or g + vec[row / T] (keys: vec = g_ksum, scal ignored).  The query's maximum takes its term at the first maximum of
 *   the features row.  gx [rows, 64] receives the diag term of the cotangent of data (the caller adds g proj).
 * u2c_qkv_gather_backward: g_q, g_k, g_v [B, H, T, 64] -> g_qkv [B, T, 3, H, 64]; normalized = 1 (pcmer_norm): g_q, g_k
 *   are cotangents of x / (|x| + 1e-8) with x read from qkv [B, T, 3, H, 64] (the forward's projection). */
int b2d_u2c_attn_readout_backward(const float* g_out, const float* out, const float* d_inv, int B, int H, int T, int dim_head,
                                  float* gn, void* stream);
int b2d_u2c_softmax_features_backward(float* g, const float* features, const float* data, const float* vec, const float* scal,
                                      int rows, int T, int n_features, int dim_head, int is_query, float eps, float* gx,
                                      void* stream);
int b2d_u2c_qkv_gather_backward(const float* g_q, const float* g_k, const float* g_v, const float* qkv, int B, int H, int T,
                                int dim_head, int normalized, float* g_qkv, void* stream);

/* ---- rectified-flow sampler of the reflow model (reflow.cu; reflow/reflow.py:51-111 around the velocity network
 * reflow/naive_v2_diff.py with conv_only and use_mlp=False): the stages between the caller's library GEMMs.  Activations
 * are token-major [B, T, C] fp32, G is a GEMM's output WITHOUT its bias.  Every output that feeds a GEMM is written as the
 * GEMM's operand: fp32 into `hi` when `lo` is NULL, else the TF32-exact halves (hi, lo) of b2d_split_tf32.  Elementwise,
 * no atomics: bit-identical from run to run.
 * rf_start: x0 [B, T, M] = t_start norm(gt) + one_minus_t_start noise with norm(v) = ((v - spec_min) / spec_range) 2 - 1,
 *   noise [B, 1, M, T] channel-major, gt [B, T, M] or NULL (then x0 = noise: also the transposing entry of a standalone
 *   velocity evaluation); x [B, T, M] receives x0 (or NULL), hi / lo its operand.
 * rf_layer_input: h [B, T, D] = GELU(G + bias) (exact erf; residual = 0) or (G + bias) + h (residual = 1), in place; then
 *   u = (h + step[b]) + cond[b, t] into hi / lo, with step row b at step + b step_stride (0: one row for every
 *   utterance) and cond row b T + t at cond + (b T + t) cond_stride; step = cond = NULL: u = h.  D, strides multiples of
 *   4, buffers 16-byte aligned.
 * rf_ode_update: v = G + bias over x [n_tokens, M].  stage -1: Euler x += v dt, emits x.  RK4 stages 0..3 with acc
 *   [n_tokens, M]: 0: acc = v, emits x + (0.5 v) dt; 1: acc += 2 v, emits x + (0.5 v) dt; 2: acc += 2 v, emits x + v dt;
 *   3: x += ((acc + v) dt) / 6, emits x.
 * rf_finish: out [n] = ((x + 1) / 2) spec_range + spec_min. */
int b2d_rf_start(const float* noise, const float* gt, float t_start, float one_minus_t_start, float spec_min,
                 float spec_range, int B, int T, int M, float* x, float* hi, float* lo, void* stream);
int b2d_rf_layer_input(const float* g, const float* bias, float* h, int residual, const float* step, int step_stride,
                       const float* cond, int cond_stride, int B, int T, int D, float* hi, float* lo, void* stream);
int b2d_rf_ode_update(const float* g, const float* bias, float* x, float* acc, int stage, float dt, int n_tokens, int M,
                      float* hi, float* lo, void* stream);
int b2d_rf_finish(const float* x, float spec_min, float spec_range, int n, float* out, void* stream);

/* ---- reflow training loss (reflow/reflow.py:20-35, :63-68, loss_type 'l2_lognorm') and the velocity network's backward
 * (reflow_bwd.cu): the stages between the caller's library GEMMs and their adjoints.  Token-major [B, T, C] fp32; G is a
 * GEMM output WITHOUT its bias.  Operand outputs (hi, lo) as above, and optional where a fp32 output is also written
 * (hi = lo = NULL: none; lo NULL: fp32 copy into hi).  No atomics: sums over tokens run per fixed slab of 32 frames of
 * one utterance into `ws` (fp64), then slab by slab in order, so results are bit-identical from run to run and do not
 * depend on the device.  `ws` is scratch of at least b2d_rf_backward_workspace_bytes(B, T, cols) bytes with cols = M
 * (rf_loss) or D n_layers (rf_layer_backward / rf_step_sums); 0 = bad shape.
 * rf_loss_input: gt [B, T, M], x0 [B, T, M] token-major, t [B] -> target = x1 - x0 with x1 = norm(gt) (as rf_start), and the
 *   operand of x_t = x0 + t_b target (fp32 products and sums in that order, no contraction) into hi / lo (hi required).
 * rf_loss: loss [1] (device) = mean over [B, T, M] of w_b (target - (G + bias[m]))^2, w [B] the per-utterance weights.
 * rf_loss_backward: gv [B, T, M] = (g_loss[0] 2 w_b / (B T M)) ((G + bias) - target), g_loss a device scalar.
 * rf_gelu_backward: gx [n_rows, C] = gy (Phi(x) + x phi(x)) with x = pre + bias[c] (bias NULL: x = pre).
 * rf_layer_backward: for layer `layer` of n_layers: gh [B T, D] += gz in place (operand into gh_hi / gh_lo); gz into
 *   columns [layer D, (layer + 1) D) of z [B T, D n_layers] (operand into z_hi / z_lo); gz's per-slab sums into ws.
 * rf_step_sums: out [B, cols] = per-utterance token sums of every column rf_layer_backward wrote into ws. */
size_t b2d_rf_backward_workspace_bytes(int B, int T, int cols);
int b2d_rf_loss_input(const float* gt, const float* x0, const float* t, float spec_min, float spec_range, int B, int T, int M,
                      float* target, float* hi, float* lo, void* stream);
int b2d_rf_loss(const float* g, const float* bias, const float* target, const float* w, int B, int T, int M, void* ws,
                size_t ws_bytes, float* loss, void* stream);
int b2d_rf_loss_backward(const float* g, const float* bias, const float* target, const float* w, const float* g_loss, int B,
                         int T, int M, float* gv, float* hi, float* lo, void* stream);
int b2d_rf_gelu_backward(const float* gy, const float* pre, const float* bias, int n_rows, int C, float* gx, float* hi,
                         float* lo, void* stream);
int b2d_rf_layer_backward(const float* gz, float* gh, int B, int T, int D, int layer, int n_layers, float* gh_hi, float* gh_lo,
                          float* z, float* z_hi, float* z_lo, void* ws, size_t ws_bytes, void* stream);
int b2d_rf_step_sums(const void* ws, size_t ws_bytes, int B, int T, int cols, float* out, void* stream);

/* ---- diffusion models' sampler (diffusion.cu; GaussianDiffusion, diffusion/diffusion.py:216-384, around the WaveNet
 * denoiser, diffusion/wavenet.py): the stages between the caller's library GEMMs.  Token-major [B, T, C] fp32, G a GEMM's
 * output WITHOUT its bias, operand outputs (hi, lo) as for rf_* above.  Elementwise, one writer per element, no atomics:
 * bit-identical from run to run.  The start and the finish are b2d_rf_start (its formula with t_start = sqrt(alpha_bar),
 * one_minus_t_start = sqrt(1 - alpha_bar) is q_sample) and b2d_rf_finish (exactly denorm_spec).
 * df_layer: stage 0: h [B T, C] = ReLU(G + bias); stage 1 / 2: r = G + bias over [B T, 2 C], h = (h + r[:C]) / sqrt 2 in
 *   place, skip [B T, C] = r[C:] (1) or skip += r[C:] (2).  Then with step (row b at step + b step_stride, 0: one row for
 *   every utterance): the k = 3 convolution's operand [B T, 3 C], row (b, t) = [y(t - 1) | y(t) | y(t + 1)] of
 *   y = h + step[b], zero outside utterance b; step NULL: skip / skip_div into the [B T, C] operand.  C and step_stride
 *   multiples of 4, buffers 16-byte aligned.
 * df_gate: z = G + cond over [n_tokens, 2 C] (cond row n at cond + n cond_stride), sigmoid(z[:C]) tanh(z[C:]) into the
 *   [n_tokens, C] operand.
 * df_relu: ReLU(G + bias) [n_tokens, C] into the operand.
 * df_update: over [B T, M]: eps = G + bias[m], d = a_x x + a_e eps, x' = c_x x + c_d d + c_1 h1 + c_2 h2 + c_3 h3 +
 *   c_n noise with coef = {a_x, a_e, c_x, c_d, c_1, c_2, c_3, c_n} (8 floats on the device); h1..h3 [B T, M] or NULL,
 *   noise [B, 1, M, T] channel-major or NULL.  d into d_out, x' into x_out and its operand into hi / lo, each optional
 *   (NULL); d_out may be one of h1..h3 and x_out may be x (element-wise in place). */
int b2d_df_layer(const float* g, const float* bias, float* h, float* skip, int stage, const float* step, int step_stride,
                 float skip_div, int B, int T, int C, float* hi, float* lo, void* stream);
int b2d_df_gate(const float* g, const float* cond, int cond_stride, int n_tokens, int C, float* hi, float* lo, void* stream);
int b2d_df_relu(const float* g, const float* bias, int n_tokens, int C, float* hi, float* lo, void* stream);
int b2d_df_update(const float* g, const float* bias, const float* coef, const float* x, float* d_out, const float* h1,
                  const float* h2, const float* h3, const float* noise, int B, int T, int M, float* x_out, float* hi,
                  float* lo, void* stream);

/* ---- diffusion training loss (diffusion/diffusion.py:194-238, q_sample + F.mse_loss, loss_type 'l2') and the WaveNet
 * denoiser's backward (diffusion_bwd.cu): the stages between the caller's library GEMMs and their adjoints.  The loss and
 * its backward are b2d_rf_loss / b2d_rf_loss_backward with w = 1 and target = noise; the step projection's cotangent is
 * b2d_rf_step_sums over the slabs df_layer_backward writes.  Token-major [B, T, C] fp32, G a GEMM output WITHOUT its
 * bias, operand outputs (hi, lo) as for rf_* above (optional where a fp32 output is also written).  No atomics, no
 * shared memory: bit-identical from run to run and independent of the device.
 * df_loss_input: the operand of x_t [B, T, M] = sqrt_ac[t_b] norm(gt) + sqrt_1m_ac[t_b] noise (norm as rf_start; fp32
 *   products and sum, no contraction), gt and noise token-major, t [B] int64 on the device, the two tables [n_steps] on
 *   the device (no host synchronisation); a t_b outside [0, n_steps) gives NaN.  hi required.
 * df_relu_backward: gx [n_rows, C] = gy where pre + bias[c] > 0, else 0.
 * df_mish_backward: gx [n] = gy mish'(x), mish(x) = x tanh(softplus(x)).
 * df_gate_backward: ga [n_tokens, C] the cotangent of df_gate's output; z = G + cond recomputed as df_gate does (cond row
 *   n at cond + n cond_stride) -> the cotangent of z [n_tokens, 2 C] into columns [layer 2 C, (layer + 1) 2 C) of
 *   gz [n_tokens, n_layers 2 C] (operand into gz_hi / gz_lo).
 * df_layer_backward: for layer `layer` of n_layers after its g_U GEMM, gu [B T, 3 C]: gh [B T, C] = gh / sqrt 2 + g_y in
 *   place with g_y(t) = gu[t + 1, block 0] + gu[t, block 1] + gu[t - 1, block 2] inside utterance b (the adjoint of
 *   df_layer's convolution operand), g_y's per-slab sums into ws (b2d_rf_backward_workspace_bytes(B, T, n_layers C)).
 *   gu NULL (the start, before the last layer): gh = 0 and ws unused.  Then gr [B T, 2 C] (optional, gsk [B T, C] then
 *   required) = [gh / sqrt 2 | gsk / skip_div], operand into gr_hi / gr_lo. */
int b2d_df_loss_input(const float* gt, const float* noise, const int64_t* t, const float* sqrt_ac, const float* sqrt_1m_ac,
                      int n_steps, float spec_min, float spec_range, int B, int T, int M, float* hi, float* lo, void* stream);
int b2d_df_relu_backward(const float* gy, const float* pre, const float* bias, int n_rows, int C, float* gx, float* hi,
                         float* lo, void* stream);
int b2d_df_mish_backward(const float* gy, const float* x, int n, float* gx, float* hi, float* lo, void* stream);
int b2d_df_gate_backward(const float* ga, const float* g, const float* cond, int cond_stride, int n_tokens, int C, int layer,
                         int n_layers, float* gz, float* gz_hi, float* gz_lo, void* stream);
int b2d_df_layer_backward(const float* gu, float* gh, const float* gsk, float skip_div, int B, int T, int C, int layer,
                          int n_layers, float* gr, float* gr_hi, float* gr_lo, void* ws, size_t ws_bytes, void* stream);

/* ---- log-mel front end of the NSF-HiFiGAN vocoder: STFT.get_mel, nsf_hifigan/nvSTFT.py:73-117 (keyshift 0, speed 1) ----
 * audio [B, n_samples] -> mel [B, n_mels, n_frames], n_frames = b2d_mel_frames(...) (0 = signal too short):
 * reflect / constant padding by (win - hop)/2, frames of win_size = n_fft = 2048 at `hop`, periodic Hann `window` [2048],
 * magnitude sqrt(re^2 + im^2 + 1e-9), mel_basis [n_mels, n_fft/2 + 1] (librosa.filters.mel layout, n_mels <= 128),
 * log(max(., clip_val)).  filter_lohi [n_mels, 2] (int32, device): first and one-past-last non-zero bin of each filter. */
int b2d_mel_frames(int n_samples, int n_fft, int win_size, int hop);
int b2d_mel_spectrogram(const float* audio, const float* window, const float* mel_basis, const int* filter_lohi, int B,
                        int n_samples, int n_fft, int win_size, int hop, int n_mels, float clip_val, float* mel, void* stream);
/* Backward of b2d_mel_spectrogram with respect to audio (training).  Same audio / tables / shape arguments as the
 * forward; bin_filter_range [n_fft/2 + 1, 2] (int32, device): first and one-past-last filter that is non-zero at each
 * bin.  grad_mel = dL/dmel, element (b, mel, frame) at grad_mel[b*grad_stride_b + mel*grad_stride_mel +
 * frame*grad_stride_frame] (elements), so the transposed [B, n_frames, n_mels] layout is read without a copy.
 * grad_audio [B, n_samples] is overwritten, deterministically (no atomics).  The mel values are recomputed bit for bit
 * as the forward computes them, so the clamp (gradient passed where mel_basis @ mag >= clip_val) matches the forward. */
int b2d_mel_spectrogram_backward(const float* audio, const float* window, const float* mel_basis, const int* filter_lohi,
                                 const int* bin_filter_range, int B, int n_samples, int n_fft, int win_size, int hop,
                                 int n_mels, float clip_val, const float* grad_mel, int64_t grad_stride_b,
                                 int64_t grad_stride_mel, int64_t grad_stride_frame, float* grad_audio, void* stream);
/* Key-shifted log-mel (STFT.get_mel with keyshift != 0, speed 1; forward only).  n_fft = n' = round(2048 *
 * 2^(keyshift / 12)) is the transform and window length, hop <= n' <= 3072 (B2D_ERR_UNSUPPORTED otherwise): padding by
 * (n' - hop)/2 as nvSTFT.py does for win_size n', periodic Hann(n') frames, the n'-point DFT's bins k < K = min(1025,
 * n'/2 + 1), magnitude sqrt(re^2 + im^2 + 1e-9) * 2048 / n' (bins K..1024 zero), the unshifted mel_basis [n_mels, 1025]
 * (n_mels <= 128) and log(max(., clip_val)) -> mel [B, n_mels, b2d_mel_frames(n_samples, n', n', hop)].
 * table: b2d_mel_keyshift_table_floats(n') floats (device, 8-byte aligned) for this n': [4, 4 + n') the window, then
 * the Bluestein chirp exp(+i pi (m^2 mod 2n') / n') at 4 + ((n' + 3) & ~3) (n' complex) and FFT_M(h) / M right after
 * it (M complex), M the smallest of 1024 / 2048 / 4096 >= n' + K - 1, h the chirp on [0, K) and mirrored on
 * (M - n', M).  Deterministic (no atomics).  Argument errors return before any CUDA call. */
int b2d_mel_keyshift_table_floats(int n_fft);
int b2d_mel_spectrogram_keyshift(const float* audio, const float* table, const float* mel_basis, const int* filter_lohi,
                                 int B, int n_samples, int n_fft, int hop, int n_mels, float clip_val, float* mel,
                                 void* stream);

/* ---- random-scale spectral loss (RSSLoss, ddsp/loss.py:9-54; the loss of configs/combsub.yaml and sins.yaml) ------------
 * Per scale n = n_ffts[s] (host array, 256 <= n <= 2047, n <= n_samples): frames of n samples at hop n (no overlap,
 * no centering), periodic Hann window w, S = |rfft(w frame)| / sqrt(sum w^2) + eps, and
 *   loss = sum_s [ mean_b ||S_t - S_p||_F / ||S_t + S_p||_F + alpha mean |log S_t - log S_p| ] / n_scale.
 * tables: host array of n_scale device pointers, each to the b2d_rss_table_floats(n) floats of that scale (8-byte
 * aligned; layout in csrc/rss_loss.cu: sqrt(sum w^2), the window, the Bluestein chirp and chirp-filter spectrum, built
 * in float64 by ddsp_svc_b200.loss.table_host).  b2d_rss_frames(n_samples, n) = 1 + (n_samples - n) / n (0 if none).
 * Forward: loss [1] fp32 and norms [n_scale, B, 2] float64 (||S_t - S_p||, ||S_t + S_p|| per scale and row) on the
 * device, through a caller-owned workspace of b2d_rss_loss_workspace_bytes (8-byte aligned); no host synchronisation,
 * no atomics, the same bits for any launch geometry.  Backward: grad_pred [B, n_samples] = grad_loss[0] * dloss/dx_pred
 * (overwritten; zero past each scale's last frame) from the forward's norms; the spectra are recomputed from x_pred and
 * x_true.  Argument errors (null pointers, misalignment, n outside [256, 2047], n_samples < n, B > 65535,
 * n_scale > 64) return B2D_ERR_* before any device call. */
int b2d_rss_table_floats(int n);
int b2d_rss_frames(int n_samples, int n);
size_t b2d_rss_loss_workspace_bytes(int B, int n_samples, int n_scale, const int* n_ffts);
int b2d_rss_loss_forward(const float* x_pred, const float* x_true, int B, int n_samples, int n_scale, const int* n_ffts,
                         const float* const* tables, float alpha, float eps, void* workspace, size_t workspace_bytes,
                         double* norms, float* loss, void* stream);
int b2d_rss_loss_backward(const float* x_pred, const float* x_true, int B, int n_samples, int n_scale, const int* n_ffts,
                          const float* const* tables, float alpha, float eps, const double* norms, const float* grad_loss,
                          float* grad_pred, void* stream);

/* ---- NSF-HiFiGAN generator (nsf_hifigan/models.py:207-273), inference (hifigan.cu) -------------------------------------
 * b2d_hifigan_conv: one Conv1d(C_in -> N, k, dilation, padding dilation (k - 1) / 2) as an implicit GEMM on the tensor
 *   cores, 3xTF32.  x element (b, t, c) at x[b x_stride_b + t x_stride_t + c x_stride_c] (token-major [B, T, C_in], or
 *   any strided view such as a channel-major mel), zero padding at each utterance's edges.  w: the weights split into
 *   TF32 (hi, lo) in mma.sync B-fragment order, [k][C_in / 8][N / 8][32 lanes][4] with lane 4 g + t holding the hi
 *   halves of W[8 nb + g, 8 kb + t, j] and W[8 nb + g, 8 kb + t + 4, j], then their lo halves
 *   (ddsp_svc_b200.hifigan.pack_conv).  lrelu != 0: leaky_relu(x, 0.1) first.
 *   up == 0: out [B, T, N] = (conv + bias[N] (+ residual) (+ accum)) / div; out may alias residual or accum.
 *   up == u > 0: the polyphase form of ConvTranspose1d(C_in, C_out = N / u, 2u, u, u / 2) (hifigan.pack_transposed):
 *   out [B, T u, C_out], element (t u + r, co) = column r C_out + co + bias[co], plus with source [B, T u noise_stride]
 *   the strided dot noise_b[co] + sum_{q < noise_k} noise_w[co, q] source[(t u + r) noise_stride - noise_pad + q]
 *   (zero outside), i.e. noise_convs[i](har_source).  k odd, C_in and N multiples of 16, C_out even, halo
 *   dilation (k - 1) / 2 <= 256; a unit channel stride needs x and its strides 16-byte aligned.
 * b2d_hifigan_post: out [B, 1, T] = tanh(bias[0] + Conv1d(C -> 1, 7, padding 3)(leaky_relu(x, 0.01))), x [B, T, C]
 *   token-major (16-byte aligned, C a multiple of 4), w [7][C] (tap-major).
 * No atomics: bit-identical from run to run. */
int b2d_hifigan_conv(const float* x, int64_t x_stride_b, int64_t x_stride_t, int64_t x_stride_c, int B, int T, int C_in,
                     const float* w, const float* bias, int k, int dilation, int N, int lrelu, const float* residual,
                     const float* accum, float div, int up, const float* source, const float* noise_w,
                     const float* noise_b, int noise_k, int noise_stride, int noise_pad, float* out, void* stream);
int b2d_hifigan_post(const float* x, const float* w, const float* bias, int B, int T, int C, float* out, void* stream);

/* b2d_sins_synth variants.  0 (default) = 1 = oscillator-bank kernel next to the impulse-response builds, then the FIR
 * kernel transforms the impulse responses itself.  2 = the bank is evaluated inside the FFT-domain FIR kernel (additionally <= 128 harmonics):
 * no [B, T] sinusoid tensor, one launch less, kept as a tested alternative (see api.cu).
 * 3 = spectrum path: a small kernel turns the impulse responses into packed 1024-point spectra once per frame (beside the
 * bank), the FIR kernel reads them: a quarter fewer transforms, 53 instead of 70 KB of shared memory (4 CTAs per SM); needs
 * block 512, both filters <= 512 taps, FIR selection 0/4; measured 4 % slower (the transform is only moved) -- the consumer
 * side of a future impulse-response GEMM that emits spectra.  Set it BEFORE querying b2d_sins_workspace_bytes (the spectra
 * live in the workspace).  All variants agree to round-off.  Process-wide test/diagnostic knob (atomic, read once per call). */
int b2d_set_sins_impl(int impl);

/* How b2d_sins_synth / b2d_combsub_synth overlap their independent kernels on an internal side stream that is joined on
 * the caller's stream before the call returns (event record/wait only; legal under stream capture).  0: every kernel on
 * the caller's stream, in order.  1: Sins: impulse-response builds next to the oscillator bank; CombSub: the dynamic-window
 * impulse response (needed by the last filter only) next to the comb source / all-pass / noise stage.  k >= 2: additionally the batch is cut into
 * k sub-batches that alternate between the two streams, staggered, so the FIR of one shares the SMs with the bank of the
 * next (-k: the same with a high-priority side stream).  Same results in every mode (the noise is keyed by the global
 * utterance index, the FFT-domain FIR is bit-identical for any batch split).  Process-wide test/diagnostic knob (atomic,
 * read once per call). */
int b2d_set_overlap(int mode);

/* Kernel selection for b2d_sinegen / b2d_source_module (measurement and A/B tests): 0 auto (= 4), 1 one sample per
 * thread (first kernel of round 1; also the only one for dim other than 1 or 9), 2 four samples per thread,
 * 3 four samples per thread with register-pair arithmetic.  Impl 1 and 2/3 draw DIFFERENT in-kernel
 * noise streams (both Philox4x32-10 keyed by seed / global utterance / position).
 * 4 = variant 2 with Philox4x32-7 instead of -10 for the in-kernel normals (7 rounds: the smallest count reported to
 * pass BigCrush; 11 % faster; Kolmogorov-Smirnov / correlation tests in tests/test_gpu_combsub_sinegen.py). */
int b2d_set_sinegen_impl(int impl);

/* ---- RMVPE pitch extractor (encoder/rmvpe/), inference (rmvpe.cu) ---------------------------------------------------
 * Activations are channel-contiguous [B, T, F, C]: element (b, t, f, c) at x[((b T + t) F + f) ld + c].
 * b2d_rmvpe_conv: a k x k convolution (k = 3: padding 1; k = 1; k = 2 with up) as an implicit GEMM on the tensor cores,
 *   3xTF32, zero padding at the T and F edges.  w: [k k][C_in / 8][N / 8][32][4] in mma.sync B-fragment order, TF32
 *   (hi, lo) halves (ddsp_svc_b200.hifigan.pack_conv of the [N, C_in, k k] weight).  out[pixel ldo + col] =
 *   act(conv + bias[col]) (+ residual[pixel ldr + col]) for col < n_valid; act 0 none, 1 relu, 2 sigmoid.  up = 1: the
 *   polyphase form of ConvTranspose2d(3x3, stride 2, padding 1, output_padding 1) (ddsp_svc_b200.rmvpe.polyphase2d):
 *   column r C_out + co (N = 4 C_out) goes to channel co of pixel (2t + r / 2, 2f + r % 2) of the [B, 2T, 2F] output,
 *   plus bias[co].  C_in and N multiples of 16, F a power of two, x and w 16-byte aligned.
 * b2d_rmvpe_conv_small: direct fp32 k x k convolution (k = 1 or 3, padding k / 2), x element (b, t, f, c) at
 *   x[b x_stride_b + t x_stride_t + f x_stride_f + c x_stride_c], optionally x in_scale[c] + in_shift[c] on every real
 *   input (before the zero padding), w [C_out][C_in][k][k], bias [C_out] or NULL, relu, C_out <= 16.  head = 0:
 *   out[pixel ldo + co]; head = 1: out[((b T + t) C_out + co) F + f] (the head's features c F + f).
 * b2d_rmvpe_pool: out [B, T / 2, F / 2, C] = AvgPool2d(2) of x (row stride ldx).
 * b2d_rmvpe_gru: the bidirectional GRU(384 -> 256) recurrence.  xg [B, T, 2][3][256] = W_ih x + b_ih of both
 *   directions (gates r, z, n), w_hh [2][768][256], b_hh [2][768] -> out [B, T, 512] = [forward | backward].  One
 *   8-CTA cluster per direction and group of 4 utterances.
 * b2d_rmvpe_resample: torchaudio Resample with the [new_freq, taps] table of ddsp_svc_b200.rmvpe.resample_table
 *   (rates divided by their gcd): out[b, j new_freq + p] = sum_k table[p, k] x[b, j orig_freq + k - width], zero
 *   outside, for the first n_out samples.
 * b2d_rmvpe_mel: log(clamp(basis @ |stft(audio, 1024, hop, hann window, center, reflect)|, 1e-5)), basis [128, 513]
 *   with lohi [128][2] the support of each row -> out [B, t_pad, 128], zeros for frames n_frames .. t_pad - 1.
 *   Needs N > 512 and n_frames = 1 + N / hop.
 * b2d_rmvpe_decode: salience [B, t_pad, 360] -> f0 [B, n_frames] (to_local_average_f0).
 * No atomics: bit-identical from run to run. */
int b2d_rmvpe_conv(const float* x, int ldx, int B, int T, int F, int C_in, const float* w, const float* bias, int k,
                   int N, int n_valid, int act, int up, const float* residual, int ldr, float* out, int ldo, void* stream);
int b2d_rmvpe_conv_small(const float* x, int64_t x_stride_b, int64_t x_stride_t, int64_t x_stride_f, int64_t x_stride_c,
                         int B, int T, int F, int C_in, const float* in_scale, const float* in_shift, const float* w,
                         const float* bias, int k, int C_out, int relu, int head, float* out, int ldo, void* stream);
int b2d_rmvpe_pool(const float* x, int ldx, int B, int T, int F, int C, float* out, void* stream);
int b2d_rmvpe_gru(const float* xg, const float* w_hh, const float* b_hh, int B, int T, float* out, void* stream);
int b2d_rmvpe_resample(const float* x, int B, int N, const float* table, int new_freq, int orig_freq, int taps,
                       int width, int n_out, float* out, void* stream);
int b2d_rmvpe_mel(const float* audio, int B, int N, const float* window, const float* basis, const int* lohi, int hop,
                  int n_frames, int t_pad, float* out, void* stream);
int b2d_rmvpe_decode(const float* salience, int B, int t_pad, int n_frames, float thred, float* f0, void* stream);

/* ---- HuBERT / ContentVec units encoder (encoder/hubert/model.py, fairseq HubertModel), inference (hubert.cu) ---------
 * Activations are token-major [B, T, C], C contiguous.  Outputs named (hi, lo) are a library GEMM's operand: fp32 into
 * `hi` when `lo` is NULL, else the TF32-exact halves of b2d_split_tf32.
 * b2d_hubert_conv0: Conv1d(1 -> 512, kernel 10, stride 5, no bias) of x [B, N] zero-padded by `pad` on the left (and
 *   as far as needed on the right) -> y [B, La, 512] for the L0 = (N + 2 pad - 10) / 5 + 1 valid frames, zeros for
 *   frames L0 .. La - 1; w [512][10].  part [B, ceil(La / 64), 2, 512] (fp64): the per-tile sums of y and y^2 over the
 *   valid frames, for b2d_hubert_gn_finalize (n_tiles = ceil(La / 64)).
 * b2d_hubert_gn_finalize: GroupNorm(512, 512) over the L0 frames -> scale, shift [B, 512] with y scale + shift the
 *   normalized, affine output.
 * b2d_hubert_act: GELU(x scale[b, c] + shift[b, c]) (the affine only when scale is non-NULL) of x [B rows_per_b, C]
 *   -> (hi, lo) of the same shape.
 * b2d_hubert_ln: row r < rows (= B T) reads x[(r / T) rows_per_b + r % T] (+ y[r] when y is non-NULL), optionally
 *   GELU, LayerNorm(C) with gamma, beta, eps -> h[r] (when non-NULL) and (hi, lo)[r] (when hi is non-NULL).  C = 512 or
 *   768; h may be x itself when rows_per_b = T.
 * b2d_hubert_posconv: y [B T, 768] = GELU(Conv1d(768, 768, 128, padding 64, groups 16)(x)[..., :T] + bias) of x
 *   [B T, 768]; w [16][128][48 in][48 out] (weight norm folded), 16-byte aligned.
 * b2d_hubert_attention: per head of qkv [B T, 2304] (q | k | v, head h at columns 64 h of each) -> (hi, lo) [B T, 768]
 *   = softmax(q k^T / 8) v, non-causal, over the T keys.
 * b2d_hubert_align: out [B, n_frames, C] = units [B, T, C] at row min(rint(ratio f), T - 1) of frame f, the product
 *   ratio f in float32 and rounded half to even.
 * No atomics: bit-identical from run to run. */
int b2d_hubert_conv0(const float* x, int B, int N, int pad, const float* w, int La, float* y, double* part,
                     void* stream);
int b2d_hubert_gn_finalize(const double* part, int B, int n_tiles, int L0, const float* gamma, const float* beta,
                           float eps, float* scale, float* shift, void* stream);
int b2d_hubert_act(const float* x, int rows, int C, int rows_per_b, const float* scale, const float* shift, float* hi,
                   float* lo, void* stream);
int b2d_hubert_ln(const float* x, const float* y, int rows, int T, int rows_per_b, int C, int gelu, const float* gamma,
                  const float* beta, float eps, float* h, float* hi, float* lo, void* stream);
int b2d_hubert_posconv(const float* x, int B, int T, const float* w, const float* bias, float* y, void* stream);
int b2d_hubert_attention(const float* qkv, int B, int T, float* hi, float* lo, void* stream);
int b2d_hubert_align(const float* units, int B, int T, int C, float ratio, int n_frames, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200DDSP_H */
