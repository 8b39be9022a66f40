"""What the offline tests share: seeded synthetic speech with pauses (no audio is stored; every case is rebuilt from
its seed), the librosa.feature.rms framing the Slicer relies on restated in float64, main.py's assembly in float64, and
main.py's / main_reflow.py's per-segment loops over this package's modules with a host round trip per segment.

The loops follow the reference line by line: each segment goes to the device from host numpy, its output comes back
with ``.cpu().numpy()`` and the result grows with ``np.append`` and the float64 ``cross_fade`` (oracle/frontend.py, a
restatement of main.py:142-149).  The f0, volume and mask are the package's kernels (checked against numpy in their own
tests), so with the same torch seed every segment sees the same inputs and draws as OfflineVC / OfflineReflowVC."""
import numpy as np

# name -> pieces of (kind, seconds): 'v' voiced (a vibrato tone with a syllable envelope, rms well above the
# Slicer's -40 dB), 's' silence (noise at -60 dB).  The Slicer's constants at 20 ms frames: min_interval 15 frames
# (0.3 s), min_length and max_sil_kept 250 frames (5 s).
SLICER_CASES = {
    "leading_silence": [("s", 6.0), ("v", 7.0)],
    "trailing_silence": [("v", 7.0), ("s", 3.0)],
    "gap_within_max_sil_kept": [("v", 6.0), ("s", 2.0), ("v", 5.0)],
    "gap_up_to_twice_max_sil_kept": [("v", 6.0), ("s", 7.5), ("v", 5.0)],
    "gap_beyond_twice_max_sil_kept": [("v", 6.0), ("s", 12.0), ("v", 4.0)],
    "gap_below_min_interval": [("v", 6.0), ("s", 0.2), ("v", 5.0)],
    "under_min_length": 200,                       # samples: the Slicer's early return counts min_length in frames
    "short_clip": [("v", 1.0), ("s", 0.5), ("v", 1.0)],
    "no_silence": [("v", 10.0)],
}
SLICER_RATES = (44100, 16000)
# the model hop split() uses at each rate (block_size * sr / sampling_rate): 512 at 44.1 kHz, 320 at 16 kHz
SPLIT_HOP = {44100: 512, 16000: 320}


def speech(pieces, sr, seed):
    """seeded synthetic speech [N] float32: the pieces one after another, or `pieces` samples of it if an int"""
    g = np.random.default_rng(seed)
    if isinstance(pieces, int):
        pieces = [("v", pieces / sr)]
    out = []
    for kind, sec in pieces:
        n = int(round(sec * sr))
        t = np.arange(n) / sr
        if kind == "v":
            f0 = g.uniform(120, 260)
            env = 0.15 * (1.2 + np.sin(2 * np.pi * g.uniform(2.5, 4.5) * t + g.uniform(0, 6)))
            phase = 2 * np.pi * np.cumsum(f0 * (1 + 0.03 * np.sin(2 * np.pi * 5 * t))) / sr
            x = env * (np.sin(phase) + 0.4 * np.sin(2 * phase + 0.3) + 0.2 * np.sin(3 * phase + 1.1))
            x = x + 0.002 * g.standard_normal(n)
        else:
            x = 0.001 * g.standard_normal(n)
        out.append(x)
    return np.concatenate(out).astype(np.float32)


def slicer_case(name, sr):
    return speech(SLICER_CASES[name], sr, seed=sorted(SLICER_CASES).index(name) * 7 + sr % 1000)


def rms64(y, frame_length, hop_length):
    """librosa.feature.rms(y=y, frame_length, hop_length) as librosa >= 0.10 computes it with center=True (zero padding
    of frame_length // 2 each side, frames of frame_length every hop_length), in float64 rounded to float32 -> [1, n]"""
    y = np.pad(np.asarray(y, dtype=np.float64), frame_length // 2)
    n = 1 + (y.shape[0] - frame_length) // hop_length
    idx = np.arange(frame_length)[None, :] + hop_length * np.arange(n)[:, None]
    return np.sqrt(np.mean(y[idx] ** 2, axis=1)).astype(np.float32)[None]


# the assembly cases: main.py's bookkeeping for the split of each slicer case at an enhancer rate other than the model's
ASSEMBLY = dict(block_size=4, model_sr=44100, out_sr=48000)


def assembly_segments(starts, stops, seed, block_size=4, model_sr=44100, out_sr=48000, short=None):
    """seeded segment outputs [float32] for these frame ranges: a little longer than their slot at out_sr, as the
    enhancer's are; ``short``: the index of one made shorter than the overlap before it (main.py's cross_fade fails)"""
    g = np.random.default_rng(seed)
    segs = []
    for i, (a, b) in enumerate(zip(starts, stops)):
        n = int(np.ceil((b - a + 1) * block_size * out_sr / model_sr)) + int(g.integers(0, 3 * block_size))
        if i == short:
            n = 2
        segs.append(g.standard_normal(n).astype(np.float32))
    return segs


def assemble64(segs, plan, total):
    """main.py's assembly at the plan's (idx, fade_len), in float64"""
    out = np.zeros(total)
    for s, (idx, fade) in zip(segs, plan):
        k = np.linspace(0, 1.0, num=fade, endpoint=True)
        out[idx:idx + fade] = (1 - k) * out[idx:idx + fade] + k * s[:fade]
        out[idx + fade:idx + s.shape[0]] = s[fade:]
    return out


# ---- main.py's and main_reflow.py's loops on the package's modules (GPU) ---------------------------------------------
def _front(vc, audio_np, sr, key, f0_min, threhold):
    import torch

    from ddsp_svc_b200 import frontend, ops
    hop = vc.hop(sr)
    x = torch.from_numpy(audio_np).to(vc.device)[None]
    f0_10 = vc.rmvpe.infer_batch(x, sr)[0]
    f0 = ops.rt_f0_regrid(f0_10.contiguous(), 0.01, audio_np.shape[0] // hop + 1, hop / sr, rmvpe=True, pad=0,
                          f0_min=float(f0_min), post_scale=2 ** (float(key) / 12))[None, :, None]
    volume = frontend.volume_extract(x, hop)
    mask = frontend.volume_mask(volume, float(threhold))
    return hop, f0, volume[..., None], mask


def _append(result, current_length, start_frame, seg_output, block_size, out_sr, model_sr):
    from oracle.frontend import cross_fade
    silent_length = round(start_frame * block_size * out_sr / model_sr) - current_length
    if silent_length >= 0:
        result = np.append(result, np.zeros(silent_length))
        result = np.append(result, seg_output)
    else:
        result = cross_fade(result, seg_output, current_length + silent_length)
    return result, current_length + silent_length + len(seg_output)


def main_loop(vc, audio_np, sr, segments, key=0, spk_id=1, spk_mix_dict=None, f0_min=50, threhold=-60,
              enhancer_adaptive_key=0):
    """main.py's loop with OfflineVC's modules -> (float64 result, out_sr, [segment outputs as float32 numpy])"""
    import torch

    from ddsp_svc_b200 import frontend
    hop, f0, volume, mask = _front(vc, audio_np, sr, key, f0_min, threhold)
    spk = torch.LongTensor(np.array([[int(spk_id)]])).to(vc.device)
    bs, msr = vc.block_size, vc.model_sr
    result, current_length, outs = np.zeros(0), 0, []
    out_sr = msr
    with torch.no_grad():
        for start_frame, end_frame in segments:
            seg_input = torch.from_numpy(audio_np[start_frame * hop:end_frame * hop]).float().unsqueeze(0).to(vc.device)
            seg_units = vc.units_encoder.encode(seg_input, sr, hop)
            seg_f0 = f0[:, start_frame:start_frame + seg_units.size(1), :]
            seg_volume = volume[:, start_frame:start_frame + seg_units.size(1), :]
            seg_output, _, _ = vc.model(seg_units, seg_f0, seg_volume, spk_id=spk, spk_mix_dict=spk_mix_dict)
            seg_output = frontend.mask_apply_(seg_output.contiguous(), mask, bs, start_frame)
            if vc.enhancer is not None:
                seg_output, out_sr = vc.enhancer.enhance(seg_output, msr, seg_f0, bs,
                                                         adaptive_key=enhancer_adaptive_key)
            seg_output = seg_output.squeeze().cpu().numpy()
            outs.append(seg_output)
            result, current_length = _append(result, current_length, start_frame, seg_output, bs, out_sr, msr)
    return result, out_sr, outs


def main_reflow_loop(vc, audio_np, sr, segments, key=0, spk_id=1, spk_mix_dict=None, f0_min=50, threhold=-60,
                     formant_shift_key=0, infer_step=2, method="euler", t_start=0.0):
    """main_reflow.py's loop with OfflineReflowVC's modules (settings already resolved) -> (float64 result, [outputs])"""
    import torch

    from ddsp_svc_b200 import frontend
    hop, f0, volume, mask = _front(vc, audio_np, sr, key, f0_min, threhold)
    spk = torch.LongTensor(np.array([[int(spk_id)]])).to(vc.device)
    aug = torch.from_numpy(np.array([[float(formant_shift_key)]])).float().to(vc.device)
    bs = vc.block_size
    result, current_length, outs = np.zeros(0), 0, []
    with torch.no_grad():
        for start_frame, end_frame in segments:
            seg_input = torch.from_numpy(audio_np[start_frame * hop:end_frame * hop]).float().unsqueeze(0).to(vc.device)
            seg_units = vc.units_encoder.encode(seg_input, sr, hop)
            seg_f0 = f0[:, start_frame:start_frame + seg_units.size(1), :]
            seg_volume = volume[:, start_frame:start_frame + seg_units.size(1), :]
            seg_output = vc.model(seg_units, seg_f0, seg_volume, spk_id=spk, spk_mix_dict=spk_mix_dict, aug_shift=aug,
                                  vocoder=vc.vocoder, infer=True, return_wav=True, infer_step=infer_step,
                                  method=method, t_start=t_start, use_tqdm=False)
            seg_output = frontend.mask_apply_(seg_output.reshape(1, -1).contiguous(), mask, bs, start_frame)
            seg_output = seg_output.squeeze().cpu().numpy()
            outs.append(seg_output)
            result, current_length = _append(result, current_length, start_frame, seg_output, bs, vc.model_sr,
                                             vc.model_sr)
    return result, outs
