"""The reflow model's cascade on the kernels: ``Unit2Wav`` and ``load_model_vocoder`` (reference reflow/vocoder.py:149-197
and :23-55), inference only.

``Unit2Wav(sampling_rate, block_size, win_length, n_unit, n_spk, use_pitch_aug, out_dims, n_layers, n_chans)`` has the
reference's parameter tree (``ddsp_model``: CombSubSuperFast; ``reflow_model``: RectifiedFlow around NaiveV2Diff), so a
reference checkpoint's ``model`` dict loads strictly.  ``forward`` follows the reference's order: the DDSP synthesizer,
the mel of its output from ``start_frame = int(silence_front * sampling_rate / block_size)`` on, the rectified-flow
sampler from ``t_start`` (skipped when ``t_start >= 1``) and, with ``return_wav``, the vocoder.

Beyond the reference, the stage's random draws can be passed in, so seeded runs compare and a CUDA graph can fill them
(session's static buffers): ``ddsp_noise`` (CombSubSuperFast's randn [B, n_frames block_size]), ``reflow_noise`` (the
sampler's [B, 1, M, T]) and SineGen's ``rand_ini`` [1, 1, 9] / ``sine_noise`` [B, T upp, 9].  Absent, each is drawn as
it is without them.

Training (``infer=False``) is not here: ``patch_reference(reflow=True)`` trains the reference's own Unit2Wav on the
kernels.
"""
import os

import torch
import torch.nn as nn
import yaml

from .dropin import DotDict
from .nsf_vocoder import Vocoder
from .reflow import NaiveV2Diff, RectifiedFlow
from .vocoder import CombSubSuperFast


def load_model_vocoder(model_path, device="cuda"):
    """config.yaml next to the checkpoint -> (Unit2Wav in eval mode with ckpt['model'] loaded strictly, its Vocoder,
    args); a model type other than 'RectifiedFlow' raises ValueError as the reference does"""
    config_file = os.path.join(os.path.split(model_path)[0], "config.yaml")
    with open(config_file, "r") as config:
        args = DotDict(yaml.safe_load(config))
    vocoder = Vocoder(args.vocoder.type, args.vocoder.ckpt, device=device)
    if args.model.type != "RectifiedFlow":
        raise ValueError(f" [x] Unknown Model: {args.model.type}")
    model = Unit2Wav(args.data.sampling_rate, args.data.block_size, args.model.win_length,
                     args.data.encoder_out_channels, args.model.n_spk, args.model.use_pitch_aug, vocoder.dimension,
                     args.model.n_layers, args.model.n_chans)
    print(" [Loading] " + model_path)
    ckpt = torch.load(model_path, map_location=torch.device(device))
    model.to(device)
    model.load_state_dict(ckpt["model"])
    model.eval()
    return model, vocoder, args


class Unit2Wav(nn.Module):
    def __init__(self, sampling_rate, block_size, win_length, n_unit, n_spk, use_pitch_aug=False, out_dims=128,
                 n_layers=6, n_chans=512):
        super().__init__()
        self.sampling_rate = sampling_rate
        self.block_size = block_size
        self.ddsp_model = CombSubSuperFast(sampling_rate, block_size, win_length, n_unit, n_spk, use_pitch_aug)
        self.reflow_model = RectifiedFlow(NaiveV2Diff(mel_channels=out_dims, dim=n_chans, num_layers=n_layers,
                                                      condition_dim=out_dims, use_mlp=False), out_dims=out_dims)

    def start_frame(self, silence_front):
        """the first DDSP frame the mel sees, the reference's way (from the model's rate)"""
        return int(silence_front * self.sampling_rate / self.block_size)

    def forward(self, units, f0, volume, spk_id=None, spk_mix_dict=None, aug_shift=None, vocoder=None, gt_spec=None,
                infer=True, return_wav=False, infer_step=10, method='euler', t_start=0.0, silence_front=0,
                use_tqdm=True, ddsp_noise=None, reflow_noise=None, rand_ini=None, sine_noise=None):
        """units [B, n_frames, n_unit], f0 / volume [B, n_frames, 1] -> the mel [B, T, M], or with ``return_wav`` the
        vocoder's audio [B, 1, T upp] (T = the mel frames from start_frame on)"""
        if not infer:
            raise NotImplementedError("Unit2Wav: training (infer=False) is not built here; patch_reference(reflow=True) "
                                      "trains the reference's Unit2Wav on the kernels")
        ddsp_wav, _, _ = self.ddsp_model(units, f0, volume, spk_id=spk_id, spk_mix_dict=spk_mix_dict,
                                         aug_shift=aug_shift, infer=infer, noise=ddsp_noise)
        start_frame = self.start_frame(silence_front)
        ddsp_mel = vocoder.extract(ddsp_wav[:, start_frame * self.block_size:]) if vocoder is not None else None
        if gt_spec is not None and ddsp_mel is None:
            ddsp_mel = gt_spec
        if t_start < 1.0:
            mel = self.reflow_model(ddsp_mel, gt_spec=ddsp_mel, infer=True, infer_step=infer_step, method=method,
                                    t_start=t_start, use_tqdm=use_tqdm, noise=reflow_noise)
        else:
            mel = ddsp_mel
        if return_wav:
            return vocoder.infer(mel, f0[:, -mel.shape[1]:], rand_ini=rand_ini, noise=sine_noise)
        return mel
