"""Drop-in for the diffusion and reflow models' ``Vocoder`` (reference diffusion/vocoder.py:80-117, the same class as
reflow/vocoder.py:58-95): the NSF-HiFiGAN mel extractor and vocoder that preprocess.py, train_diff.py, main_diff.py
and main_reflow.py build from ``args.vocoder.type`` / ``args.vocoder.ckpt``.

``Vocoder(vocoder_type, vocoder_ckpt, device=None)`` reads the checkpoint's config.json ('nsf-hifigan', or
'nsf-hifigan-log10', whose mels are scaled by 0.434294 before vocoding) and exposes ``vocoder_sample_rate``,
``vocoder_hop_size`` and ``dimension`` as the reference does.

- ``extract(audio [B, T], sample_rate=0, keyshift=0) -> [B, n_frames, n_mels]``: resampling to the vocoder's rate on
  the kernels (rmvpe.Resampler, torchaudio's lowpass_filter_width=128 table), then ``mel.STFT.get_mel`` for keyshift 0
  (differentiable with respect to audio: the DDSP loss keeps its CUDA backward) or ``get_mel_keyshift`` otherwise
  (forward only).  Resampling has no backward: under grad with an audio that requires grad it raises.
- ``infer(mel [B, n_frames, n_mels], f0 [B, >= n_frames, 1], rand_ini=None, noise=None) -> audio``: the package's
  NSF-HiFiGAN ``Generator``, built on first use from config.json and ``ckpt['generator']`` as
  nsf_hifigan.models.load_model builds it, with torch's CPU generator restored after the build (SineGen's noise seed
  comes from it, so the first call draws what later calls draw under the same seed).  ``rand_ini`` [1, 1, 9] /
  ``noise`` [B, n_frames upp, 9] (not in the reference) take SineGen's draws, for seeded runs and CUDA graphs; without
  them it draws as the reference does.
"""
import json
import os

import torch

from .mel import STFT
from .rmvpe import Resampler

LOG10_SCALE = 0.434294


def load_config(model_path):
    """config.json next to the checkpoint, as nsf_hifigan.models.load_config reads it (attribute access)"""
    from .dropin import DotDict
    with open(os.path.join(os.path.split(model_path)[0], "config.json")) as f:
        return DotDict(json.load(f))


def load_generator(model_path, device):
    """nsf_hifigan.models.load_model on the package's Generator: config.json, ckpt['generator'], eval, weight norm
    removed -> (generator, h)"""
    from .hifigan import Generator
    h = load_config(model_path)
    generator = Generator(h).to(device)
    cp_dict = torch.load(model_path, map_location=device)
    generator.load_state_dict(cp_dict["generator"])
    generator.eval()
    generator.remove_weight_norm()
    return generator, h


class Vocoder:
    def __init__(self, vocoder_type, vocoder_ckpt, device=None):
        if vocoder_type not in ("nsf-hifigan", "nsf-hifigan-log10"):
            raise ValueError(f" [x] Unknown vocoder: {vocoder_type}")
        device = torch.device("cuda" if device is None else device)
        if device.type != "cuda":
            raise ValueError("the vocoder runs on the CUDA kernels: device must be a CUDA device, got %s" % device)
        self.device = device
        self.vocoder_type = vocoder_type
        self.model_path = vocoder_ckpt
        self.model = None
        h = self.h = load_config(vocoder_ckpt)
        self.stft = STFT(h.sampling_rate, h.num_mels, h.n_fft, h.win_size, h.hop_size, h.fmin, h.fmax)
        self._resampler = Resampler(h.sampling_rate)
        self.resample_kernel = self._resampler.tables
        self.vocoder_sample_rate = h.sampling_rate
        self.vocoder_hop_size = h.hop_size
        self.dimension = h.num_mels

    def extract(self, audio, sample_rate=0, keyshift=0):
        if sample_rate == self.vocoder_sample_rate or sample_rate == 0:
            audio_res = audio
        else:
            if torch.is_grad_enabled() and isinstance(audio, torch.Tensor) and audio.requires_grad:
                raise NotImplementedError("resampling has no backward on the kernels: pass audio at %d Hz (or "
                                          "sample_rate=0) when the mel must be differentiable" % self.vocoder_sample_rate)
            if not (isinstance(audio, torch.Tensor) and audio.is_cuda and audio.dim() == 2):
                raise ValueError("audio must be a [B, T] CUDA tensor")
            audio_res = self._resampler(audio.float().contiguous(), sample_rate)
        if keyshift == 0:
            m = self.stft.get_mel(audio_res)
        else:
            m = self.stft.get_mel_keyshift(audio_res, keyshift)
        return m.transpose(1, 2)                            # B, n_frames, bins

    def infer(self, mel, f0, rand_ini=None, noise=None):
        f0 = f0[:, :mel.size(1), 0]                         # B, n_frames
        if self.model is None:
            print('| Load HifiGAN: ', self.model_path)
            # the modules' default init draws from torch's CPU generator, which also seeds SineGen's noise below: a
            # forked generator keeps the first call's draws those of every later call under the same seed
            with torch.random.fork_rng(devices=[]):
                self.model, self.h = load_generator(self.model_path, self.device)
        with torch.no_grad():
            c = mel.transpose(1, 2)
            if self.vocoder_type == "nsf-hifigan-log10":
                c = LOG10_SCALE * c
            draws = {k: v for k, v in (("rand_ini", rand_ini), ("noise", noise)) if v is not None}
            return self.model(c, f0, **draws)
