"""CPU restatement of the reference synthesis path with the reference's own ATen operators.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py) -- never imported by the product.

Why torch: the arithmetic of this path does not live in the reference at all, it
lives in PyTorch's CPU kernels (upsample_linear1d, cumsum with fp64 accumulation,
sin, pocketfft rfft/irfft/stft/istft, col2im, mt19937).  PyTorch is an unpinned
third-party dependency of the reference (requirements.txt lists no torch; README
names 1.9.1 / 2.0.0); the build container and the GPU box both carry torch 2.11.0.
Restating the algorithm on the same operators makes this port bit-identical to the
live reference on CPU, which tests/test_oracle_vs_reference.py checks whenever
the reference is importable, and tests/test_oracle_golden.py checks against vectors
the live reference produced (tests/golden/make_golden.py).

Every function returns the intermediate stage outputs as well, so the CUDA path can
be compared stage by stage.  All inputs are CPU tensors; ``ctrls`` are the RAW
(pre-activation) Unit2Control outputs.
"""
import math

import torch
import torch.nn.functional as F

TWO_PI = 2 * math.pi


# --------------------------------------------------------------------------------------
# frame -> sample interpolation            (reference ddsp/core.py:66-70  `upsample`)
# --------------------------------------------------------------------------------------
def frames_to_samples(v, block):
    """[B, nF, C] -> [B, nF*block, C]; linear, last frame held (v[nF] := v[nF-1])."""
    n_frames = v.shape[1]
    ch_first = v.transpose(1, 2)
    padded = torch.cat((ch_first, ch_first[:, :, -1:]), dim=2)
    up = F.interpolate(padded, size=n_frames * block + 1, mode="linear", align_corners=True)
    return up[:, :, :-1].transpose(1, 2)


# --------------------------------------------------------------------------------------
# exciter phase                 (reference ddsp/vocoder.py:564-575, :743-753, :819-829)
# --------------------------------------------------------------------------------------
def wrapped_phase(f0_frames, sampling_rate, block, initial_phase=None, infer=True):
    """Returns (x, f0_up): x = wrapped phase in CYCLES, fp32, [B, T, 1]."""
    sr = torch.tensor(sampling_rate)
    f0_up = frames_to_samples(f0_frames, block)
    if infer:
        acc = torch.cumsum(f0_up.double() / sr, dim=1)
    else:
        acc = torch.cumsum(f0_up / sr, dim=1)
    if initial_phase is not None:
        acc = acc + initial_phase.to(acc) / 2 / math.pi
    acc = acc - torch.round(acc)
    return acc.to(f0_up), f0_up


# --------------------------------------------------------------------------------------
# control activations   (reference ddsp/vocoder.py:580-585, ddsp/core.py:73-77)
# --------------------------------------------------------------------------------------
def harmonic_amplitudes(c_amp, f0_frames, sampling_rate):
    amp = torch.exp(c_amp) / 128
    n_h = amp.shape[-1]
    harm_hz = f0_frames * torch.arange(1, n_h + 1).to(f0_frames)
    keep = (harm_hz < (torch.tensor(sampling_rate) / 2)).float() + 1e-7
    return amp * keep


# --------------------------------------------------------------------------------------
# additive bank                                  (reference ddsp/vocoder.py:586-594)
# --------------------------------------------------------------------------------------
def sinusoid_bank(x_cycles, amp_frames, block, chunk=32):
    phase = TWO_PI * x_cycles
    n_h = amp_frames.shape[-1]
    order = torch.arange(1, n_h + 1).to(phase)
    out = 0.0
    for lo in range(0, n_h, chunk):
        hi = lo + chunk
        out = out + (torch.sin(phase * order[lo:hi])
                     * frames_to_samples(amp_frames[:, :, lo:hi], block)).sum(-1)
    return out


# --------------------------------------------------------------------------------------
# impulse responses          (reference ddsp/core.py:254-270, :185-237, :240-251)
# --------------------------------------------------------------------------------------
def impulse_response(spectrum, window="none", half_width_frames=None):
    """spectrum [B, nF, M] complex64 -> causal-form IR [B, nF, 2(M-1)] fp32.

    window: "none" (roll only), "hann" (static periodic Hann), "dynamic" (per-frame
    raised cosine of half-width ``half_width_frames`` [B, nF, 1]).
    """
    ir = torch.fft.irfft(spectrum)
    size = ir.shape[-1]
    if window == "none":
        return ir.roll(size // 2, -1)
    if window == "hann":
        w = torch.hann_window(size).to(ir)
        w = w.roll(size // 2, -1).unsqueeze(0)
        return (ir * w).roll(size // 2, -1)
    if window == "dynamic":
        w = torch.arange(-(size // 2), (size + 1) // 2).to(ir) / half_width_frames
        w[w > 1] = 0
        w = (1 + torch.cos(math.pi * w)) / 2
        return ir.roll(size // 2, -1) * w
    raise ValueError(window)


# --------------------------------------------------------------------------------------
# time-varying FIR by overlap-add                (reference ddsp/core.py:120-182)
# --------------------------------------------------------------------------------------
def ltv_fir(audio, ir):
    """audio [B, T], ir [B, nF, L] -> [B, T]."""
    n_batch, n_frames, taps = ir.shape
    if audio.shape[0] != n_batch:
        raise ValueError("Batch size of audio ({}) and impulse response ({}) must be the same."
                         .format(audio.shape[0], n_batch))
    n_samples = audio.shape[1]
    hop = int(n_samples / n_frames)
    span = 2 * hop
    frames = F.pad(audio, (hop, hop)).unfold(1, span, hop)
    frames = frames * torch.bartlett_window(span).to(frames)
    n_fft = taps + span - 1
    spec = torch.fft.rfft(frames, n_fft)
    ir_all = torch.cat((ir, ir[:, -1:, :]), dim=1)
    spec = spec * torch.fft.rfft(ir_all, n_fft)
    pieces = torch.fft.irfft(spec, n_fft)
    n_pieces, piece_len = pieces.shape[1], pieces.shape[2]
    ola = torch.nn.Fold(output_size=(1, (n_pieces - 1) * hop + piece_len),
                        kernel_size=(1, piece_len), stride=(1, hop))
    full = ola(pieces.transpose(1, 2)).squeeze(1).squeeze(1)[:, hop:]
    start = taps // 2
    end = (full.shape[-1] - n_samples) - start
    return full[:, start:-end]


# --------------------------------------------------------------------------------------
# Sins                                           (reference ddsp/vocoder.py:556-611)
# --------------------------------------------------------------------------------------
def sins_forward(f0_frames, ctrls, sampling_rate, block, noise=None, initial_phase=None,
                 infer=True, chunk=32):
    x, _ = wrapped_phase(f0_frames, sampling_rate, block, initial_phase, infer)
    phase_frames = (TWO_PI * x)[:, ::block, :]
    amp = harmonic_amplitudes(ctrls["amplitudes"], f0_frames, sampling_rate)
    group_delay = math.pi * torch.tanh(ctrls["group_delay"])
    noise_mag = torch.exp(ctrls["noise_magnitude"]) / 128
    sinusoids = sinusoid_bank(x, amp, block, chunk)
    ir_allpass = impulse_response(torch.exp(1.j * torch.cumsum(group_delay, dim=-1)), "none")
    harmonic = ltv_fir(sinusoids, ir_allpass)
    if noise is None:
        noise = torch.rand_like(harmonic) * 2 - 1
    ir_noise = impulse_response(torch.complex(noise_mag, torch.zeros_like(noise_mag)), "hann")
    noise_out = ltv_fir(noise, ir_noise)
    return {"x": x, "phase_frames": phase_frames, "sinusoids": sinusoids,
            "ir_allpass": ir_allpass, "ir_noise": ir_noise, "noise_in": noise,
            "harmonic": harmonic, "noise": noise_out, "signal": harmonic + noise_out}


# --------------------------------------------------------------------------------------
# CombSub (old)                                  (reference ddsp/vocoder.py:811-862)
# --------------------------------------------------------------------------------------
def combsub_forward(f0_frames, ctrls, sampling_rate, block, noise=None, initial_phase=None,
                    infer=True):
    sr = torch.tensor(sampling_rate)
    x, f0_up = wrapped_phase(f0_frames, sampling_rate, block, initial_phase, infer)
    phase_frames = TWO_PI * x[:, ::block, :]
    group_delay = math.pi * torch.tanh(ctrls["group_delay"])
    src_mag = torch.exp(ctrls["harmonic_magnitude"])
    noise_mag = torch.exp(ctrls["noise_magnitude"]) / 128
    comb = torch.sinc(sr * x / (f0_up + 1e-3)).squeeze(-1)
    ir_allpass = impulse_response(torch.exp(1.j * torch.cumsum(group_delay, dim=-1)), "none")
    allpassed = ltv_fir(comb, ir_allpass)
    ir_harm = impulse_response(torch.complex(src_mag, torch.zeros_like(src_mag)), "dynamic",
                               1.5 * sr / (f0_frames + 1e-3))
    harmonic = ltv_fir(allpassed, ir_harm)
    if noise is None:
        noise = torch.rand_like(harmonic) * 2 - 1
    ir_noise = impulse_response(torch.complex(noise_mag, torch.zeros_like(noise_mag)), "hann")
    noise_out = ltv_fir(noise, ir_noise)
    return {"x": x, "phase_frames": phase_frames, "comb": comb, "ir_allpass": ir_allpass,
            "allpassed": allpassed, "ir_harmonic": ir_harm, "ir_noise": ir_noise,
            "noise_in": noise, "harmonic": harmonic, "noise": noise_out,
            "signal": harmonic + noise_out}


# --------------------------------------------------------------------------------------
# CombSubSuperFast                               (reference ddsp/vocoder.py:639-710)
# --------------------------------------------------------------------------------------
def superfast_source(f0_frames, sampling_rate, block):
    """Closed-form comb-tooth source (reference fast_source_gen, ddsp/vocoder.py:639-651)."""
    sr = torch.tensor(sampling_rate)
    j = torch.arange(block)
    s = f0_frames / sr
    ds = F.pad(s[:, 1:, :] - s[:, :-1, :], (0, 0, 0, 1))
    rad = s * (j + 1) + 0.5 * ds * j * (j + 1) / block
    s_up = s + ds * j / block
    adv = torch.fmod(rad[..., -1:].float() + 0.5, 1.0) - 0.5
    acc = adv.cumsum(dim=1).fmod(1.0).to(f0_frames)
    rad = rad + F.pad(acc[:, :-1, :], (0, 0, 1, 0))
    rad = rad - torch.round(rad)
    comb = torch.sinc(rad / (s_up + 1e-5)).reshape(f0_frames.shape[0], -1)
    return comb, TWO_PI * rad[:, :, :1]


def superfast_forward(f0_frames, ctrls, sampling_rate, block, win_length, noise=None):
    window = torch.hann_window(win_length)
    comb, phase_frames = superfast_source(f0_frames, sampling_rate, block)
    hold_last = lambda z: torch.cat((z, z[:, -1:, :]), dim=1)
    h_src = hold_last(torch.exp(ctrls["harmonic_magnitude"] + 1.j * math.pi * ctrls["harmonic_phase"]))
    h_noise = hold_last(torch.exp(ctrls["noise_magnitude"] + 1.j * math.pi * ctrls["noise_phase"]) / 128)
    pad_mode = "reflect" if comb.shape[-1] > win_length // 2 else "constant"
    stft = lambda z: torch.stft(z, n_fft=win_length, win_length=win_length, hop_length=block,
                                window=window, center=True, return_complex=True, pad_mode=pad_mode)
    if noise is None:
        noise = torch.randn_like(comb)
    spec = stft(comb) * h_src.permute(0, 2, 1) + stft(noise) * h_noise.permute(0, 2, 1)
    signal = torch.istft(spec, n_fft=win_length, win_length=win_length, hop_length=block,
                         window=window, center=True)
    return {"comb": comb, "phase_frames": phase_frames, "noise_in": noise, "signal": signal}


# --------------------------------------------------------------------------------------
# CombSubFast                                    (reference ddsp/vocoder.py:735-786)
# --------------------------------------------------------------------------------------
def combsubfast_forward(f0_frames, ctrls, sampling_rate, block, noise=None, initial_phase=None, infer=True):
    """sqrt-Hann analysis/synthesis frames of 2*block at hop block; per-frame complex source filter and real
    noise filter applied in the rfft domain; plain overlap-add (sqrt-Hann^2 is COLA at 50 % overlap)."""
    sr = torch.tensor(sampling_rate)
    x, f0_up = wrapped_phase(f0_frames, sampling_rate, block, initial_phase, infer)       # (:743-751)
    phase_frames = TWO_PI * x[:, ::block, :]                                              # (:753)
    hold_last = lambda z: torch.cat((z, z[:, -1:, :]), dim=1)
    h_src = hold_last(torch.exp(ctrls["harmonic_magnitude"] + 1.j * math.pi * ctrls["harmonic_phase"]))   # (:758-759)
    h_noise = hold_last(torch.exp(ctrls["noise_magnitude"]) / 128)                        # (:760-761)
    comb = torch.sinc(sr * x / (f0_up + 1e-3)).squeeze(-1)                                # (:764-765)
    n_fft = 2 * block
    window = torch.sqrt(torch.hann_window(n_fft))                                         # (:726)
    frames_of = lambda z: F.pad(z, (block, block)).unfold(1, n_fft, block) * window       # (:766-767, :772-773)
    if noise is None:
        noise = torch.rand_like(comb) * 2 - 1                                             # (:771)
    spec = torch.fft.rfft(frames_of(comb), n_fft) * h_src + torch.fft.rfft(frames_of(noise), n_fft) * h_noise   # (:768-777)
    pieces = torch.fft.irfft(spec, n_fft) * window                                        # (:780)
    ola = torch.nn.Fold(output_size=(1, (pieces.size(1) + 1) * block), kernel_size=(1, n_fft), stride=(1, block))
    signal = ola(pieces.transpose(1, 2))[:, 0, 0, block:-block]                           # (:783-784)
    return {"x": x, "phase_frames": phase_frames, "comb": comb, "noise_in": noise, "signal": signal}


# --------------------------------------------------------------------------------------
# SineGen                                        (reference nsf_hifigan/models.py:134-165)
# --------------------------------------------------------------------------------------
def sinegen_forward(f0, upp, sampling_rate, harmonic_num=8, sine_amp=0.1, noise_std=0.003,
                    voiced_threshold=0, rand_ini=None, noise=None):
    """f0 [B, nF] -> [B, nF*upp, harmonic_num+1].  RNG draw order when not given explicitly:
    first rand(1,1,dim) for the initial phases, then randn_like for the additive noise."""
    dim = harmonic_num + 1
    f0 = f0.unsqueeze(-1)
    rad = f0 / sampling_rate * torch.arange(1, upp + 1)
    adv = torch.fmod(rad[..., -1:].float() + 0.5, 1.0) - 0.5
    acc = adv.cumsum(dim=1).fmod(1.0).to(f0)
    rad = rad + F.pad(acc, (0, 0, 1, -1))
    rad = rad.reshape(f0.shape[0], -1, 1) * torch.arange(1, dim + 1).reshape(1, 1, -1)
    if rand_ini is None:
        rand_ini = torch.rand(1, 1, dim)
        rand_ini[..., 0] = 0
    rad = rad + rand_ini
    sines = torch.sin(TWO_PI * rad) * sine_amp
    uv = (f0 > voiced_threshold).float()
    uv = F.interpolate(uv.transpose(2, 1), scale_factor=upp, mode="nearest").transpose(2, 1)
    noise_amp = uv * noise_std + (1 - uv) * sine_amp / 3
    if noise is None:
        noise = torch.randn_like(sines)
    return {"rand_ini": rand_ini, "noise_in": noise, "out": sines * uv + noise_amp * noise}


# ------------------------------------------------------------------------------------------
# SourceModuleHnNSF tail                          (reference nsf_hifigan/models.py:201-204)
# ------------------------------------------------------------------------------------------
def source_module_forward(f0, upp, sampling_rate, weight, bias, harmonic_num=8, **kw):
    """sine_merge = tanh(l_linear(sine_wavs)): [B, T, 1].  ``weight`` [1, dim], ``bias`` [1]."""
    sines = sinegen_forward(f0, upp, sampling_rate, harmonic_num, **kw)["out"]          # (:202)
    return {"out": torch.tanh(torch.nn.functional.linear(sines, weight, bias)), "sines": sines}   # (:203)
