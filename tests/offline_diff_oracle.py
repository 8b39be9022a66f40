"""main_diff.py's loop and batch_infer.py's infer() over OfflineDiffVC's modules (GPU), for
tests/test_gpu_offline_diff.py and bench_offline_diff.py.

Both follow the reference line by line with the settings already resolved (``offline.diff_settings``, checked against
the drivers' own lines in tests/test_offline_diff.py): the speaker ids and the formant key go to the device from host
numpy, the input's mel gets its last frame repeated, each segment goes to the device from host numpy and its output
comes back with ``.cpu().numpy()``, and the result grows with ``np.append`` and the float64 ``cross_fade``
(offline_oracle._append).  The f0, volume and mask are the package's kernels (offline_oracle._front), so with the same
torch seed every model call sees the same inputs and draws as OfflineDiffVC's."""
import numpy as np

from tests.offline_oracle import _append, _front


def _ids(vc, s, spk_id, formant_shift_key):
    import torch
    spk_id = torch.LongTensor(np.array([[int(spk_id)]])).to(vc.device)
    diff_spk_id = spk_id if s.diff_spk_id is None else torch.LongTensor(np.array([[int(s.diff_spk_id)]])).to(vc.device)
    formant = torch.from_numpy(np.array([[float(formant_shift_key)]])).float().to(vc.device)
    return spk_id, diff_spk_id, formant


def _input_mel(vc, audio_np, sr):
    import torch
    audio_t = torch.from_numpy(audio_np).float().unsqueeze(0).to(vc.device)
    input_mel = vc.vocoder.extract(audio_t, sr)
    return torch.cat((input_mel, input_mel[:, -1:, :]), 1)


def main_diff_loop(vc, audio_np, sr, segments, s, key=0, spk_id=1, spk_mix_dict=None, f0_min=50, threhold=-60,
                   formant_shift_key=0):
    """main_diff.py:344-388 with OfflineDiffVC's modules and the settings ``s`` -> (float64 result, [segment outputs as
    float32 numpy])"""
    import torch

    from ddsp_svc_b200 import frontend
    hop, f0, volume, mask = _front(vc, audio_np, sr, key, f0_min, threhold)
    spk_id, diff_spk_id, formant = _ids(vc, s, spk_id, formant_shift_key)
    ddsp = vc.ddsp_model if s.mode == "ddsp" else None
    input_mel = _input_mel(vc, audio_np, sr) if s.mode == "input_mel" else None
    bs, msr = vc.block_size, vc.model_sr
    result, current_length, outs = np.zeros(0), 0, []
    with torch.no_grad():
        for start_frame, end_frame in segments:
            seg_input = torch.from_numpy(audio_np[start_frame * hop:end_frame * hop]).float().unsqueeze(0).to(vc.device)
            seg_units = vc.units_encoder.encode(seg_input, sr, hop)
            seg_f0 = f0[:, start_frame:start_frame + seg_units.size(1), :]
            seg_volume = volume[:, start_frame:start_frame + seg_units.size(1), :]
            if ddsp is not None:
                seg_ddsp_f0 = 2 ** (-float(formant_shift_key) / 12) * seg_f0
                seg_ddsp_output, _, (_, _) = ddsp(seg_units, seg_ddsp_f0, seg_volume, spk_id=spk_id,
                                                  spk_mix_dict=spk_mix_dict)
                seg_input_mel = vc.vocoder.extract(seg_ddsp_output, msr, keyshift=float(formant_shift_key))
            elif input_mel is not None:
                seg_input_mel = input_mel[:, start_frame:start_frame + seg_units.size(1), :]
            else:
                seg_input_mel = None
            seg_mel = vc.model(seg_units, seg_f0, seg_volume, spk_id=diff_spk_id, spk_mix_dict=spk_mix_dict,
                               aug_shift=formant, vocoder=vc.vocoder, gt_spec=seg_input_mel, infer=True,
                               infer_speedup=s.infer_speedup, method=s.method, k_step=s.k_step, use_tqdm=False)
            seg_output = vc.vocoder.infer(seg_mel, seg_f0)
            seg_output = frontend.mask_apply_(seg_output.reshape(1, -1).contiguous(), mask, bs, start_frame)
            seg_output = seg_output.squeeze().cpu().numpy()
            outs.append(seg_output)
            result, current_length = _append(result, current_length, start_frame, seg_output, bs, msr, msr)
    return result, outs


def batch_infer(vc, audio_np, sr, s, key=0, spk_id=1, spk_mix_dict=None, f0_min=50, threhold=-60,
                formant_shift_key=0):
    """batch_infer.py's infer() (:270-363) with OfflineDiffVC's modules and the settings ``s`` -> float32 numpy
    [n_frames block_size]"""
    import torch

    from ddsp_svc_b200 import frontend
    hop, f0, volume, mask = _front(vc, audio_np, sr, key, f0_min, threhold)
    formant_shift_key_t = torch.from_numpy(np.array([[float(formant_shift_key)]])).float().to(vc.device)
    input = torch.from_numpy(audio_np).float().unsqueeze(0).to(vc.device)
    units = vc.units_encoder.encode(input, sr, hop)
    spk_id, diff_spk_id, _ = _ids(vc, s, spk_id, formant_shift_key)
    input_mel = _input_mel(vc, audio_np, sr) if s.mode == "input_mel" else None
    ddsp = vc.ddsp_model if s.mode == "ddsp" else None
    with torch.no_grad():
        if ddsp is not None:
            ddsp_f0 = 2 ** (-float(formant_shift_key) / 12) * f0
            ddsp_output, _, (_, _) = ddsp(units, ddsp_f0, volume, spk_id=spk_id, spk_mix_dict=spk_mix_dict)
            input_mel = vc.vocoder.extract(ddsp_output, vc.model_sr, keyshift=float(formant_shift_key))
        mel = vc.model(units, f0, volume, spk_id=diff_spk_id, spk_mix_dict=spk_mix_dict,
                       aug_shift=formant_shift_key_t, vocoder=vc.vocoder,
                       gt_spec=input_mel[:, :units.size(1)] if input_mel is not None else None, infer=True,
                       infer_speedup=s.infer_speedup, method=s.method, k_step=s.k_step, use_tqdm=False)
        output = vc.vocoder.infer(mel, f0)
        output = frontend.mask_apply_(output.reshape(1, -1).contiguous(), mask, vc.block_size, 0)
        return output.squeeze().cpu().numpy()
