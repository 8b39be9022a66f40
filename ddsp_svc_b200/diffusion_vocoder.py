"""The diffusion models' cascade on the kernels: ``Unit2Mel``, ``Unit2Wav``, ``Unit2WavFast`` and ``load_model_vocoder``
(reference diffusion/vocoder.py:24-78 and :171-314), and ``DiffGtMel`` (diffusion/infer_gt_mel.py), inference only.

- ``Unit2Mel`` ('Diffusion', configs/diffusion.yaml): the condition ``unit_embed(units) + f0_embed(log(1 + f0/700)) +
  volume_embed(volume)`` (+ the speaker row or mix, + ``aug_shift_embed(aug_shift / 5)``) feeds GaussianDiffusion around
  WaveNet.  unit_embed is one library GEMM at ``gemm_precision`` (unit2control._Gemm, "3xtf32" by default) and the rest
  is the b2d_u2c_embed kernel without its phase term, in the reference's association.  The speaker row (or the mix's
  sum) is built from the embedding weight with host integers, so nothing is copied to the device.
- ``Unit2Wav`` ('DiffusionNew'): CombSubFast, the mel of its output, GaussianDiffusion(WaveNet) conditioned on the
  synthesizer's hidden state.
- ``Unit2WavFast`` ('DiffusionFast'): CombSubSuperFast, the mel of its output, GaussianDiffusion(NaiveV2Diff)
  conditioned on that mel.

Each has the reference's parameter tree and buffers, so a reference checkpoint's ``model`` dict loads strictly, and its
``forward`` follows the reference line by line.  Beyond the reference, every random draw can be passed in, so seeded
runs compare and a CUDA graph can fill them from static buffers: ``ddsp_noise`` (the synthesizer's noise, [B, n_frames
block_size]), ``noise`` (the sampler's start, [B, 1, M, T], any strides), ``step_noise`` (DDPM's per-step draws) and
SineGen's ``rand_ini`` [1, 1, 9] / ``sine_noise`` [B, T upp, 9].  Absent, each is drawn as it is without them.

Training (``infer=False``) is not here: ``patch_reference(diffusion=True)`` trains the reference's own models on the
kernels.
"""
import os

import torch
import torch.nn as nn
import torch.nn.functional as F
import yaml

from . import _lib
from .diffusion import GaussianDiffusion, WaveNet
from .dropin import DotDict
from .nsf_vocoder import Vocoder
from .ops import _need_cuda_f32, _stream
from .reflow import NaiveV2Diff
from .unit2control import _Gemm, _k, _split
from .vocoder import CombSubFast, CombSubSuperFast

_TRAINING = ("%s: training (infer=False) is not built here; patch_reference(diffusion=True) trains the reference's "
             "%s on the kernels")


def read_config(model_path):
    """config.yaml next to the checkpoint, with attribute access"""
    with open(os.path.join(os.path.split(model_path)[0], "config.yaml"), "r") as config:
        return DotDict(yaml.safe_load(config))


def build_model(args, out_dims):
    """the model of ``args.model.type`` ('Diffusion', 'DiffusionNew', 'DiffusionFast'); another type raises ValueError
    as the reference does"""
    if args.model.type == "Diffusion":
        return Unit2Mel(args.data.encoder_out_channels, args.model.n_spk, args.model.use_pitch_aug, out_dims,
                        args.model.n_layers, args.model.n_chans, args.model.n_hidden)
    if args.model.type == "DiffusionNew":
        return Unit2Wav(args.data.sampling_rate, args.data.block_size, args.data.encoder_out_channels, args.model.n_spk,
                        args.model.use_pitch_aug, out_dims, args.model.n_layers, args.model.n_chans,
                        pcmer_norm=args.model.pcmer_norm)
    if args.model.type == "DiffusionFast":
        return Unit2WavFast(args.data.sampling_rate, args.data.block_size, args.model.win_length,
                            args.data.encoder_out_channels, args.model.n_spk, args.model.use_pitch_aug, out_dims,
                            args.model.n_layers, args.model.n_chans)
    raise ValueError(f" [x] Unknown Model: {args.model.type}")


def load_model_vocoder(model_path, device="cuda"):
    """config.yaml next to the checkpoint -> (the model in eval mode with ckpt['model'] loaded strictly, its Vocoder,
    args)"""
    args = read_config(model_path)
    vocoder = Vocoder(args.vocoder.type, args.vocoder.ckpt, device=device)
    model = build_model(args, vocoder.dimension)
    print(" [Loading] " + model_path)
    ckpt = torch.load(model_path, map_location=torch.device(device))
    model.to(device)
    model.load_state_dict(ckpt["model"])
    model.eval()
    return model, vocoder, args


class Unit2Mel(nn.Module):
    #: precision of the unit_embed GEMM, see unit2control._Gemm: "3xtf32" (default), "fp32", "tf32"
    gemm_precision = "3xtf32"

    def __init__(self, input_channel, n_spk, use_pitch_aug=False, out_dims=128, n_layers=20, n_chans=384,
                 n_hidden=256):
        super().__init__()
        if n_hidden != 256:
            raise ValueError("Unit2Mel: n_hidden must be 256 (the condition's embed kernel is 256 wide; every "
                             "configuration builds 256), got %r" % (n_hidden,))
        self.unit_embed = nn.Linear(input_channel, n_hidden)
        self.f0_embed = nn.Linear(1, n_hidden)
        self.volume_embed = nn.Linear(1, n_hidden)
        if use_pitch_aug:
            self.aug_shift_embed = nn.Linear(1, n_hidden, bias=False)
        else:
            self.aug_shift_embed = None
        self.n_spk = n_spk
        if n_spk is not None and n_spk > 1:
            self.spk_embed = nn.Embedding(n_spk, n_hidden)
        self.decoder = GaussianDiffusion(WaveNet(out_dims, n_layers, n_chans, n_hidden), out_dims=out_dims)
        self.__dict__["_packed"] = None

    def _pack(self):
        """unit_embed's weight as the GEMM wants it and the embed kernel's [7, 256] table (f0 w, f0 b, two unused phase
        rows, volume w, volume b, aug w), rebuilt when a parameter changes"""
        params = (self.unit_embed.weight, self.unit_embed.bias, self.f0_embed.weight, self.f0_embed.bias,
                  self.volume_embed.weight, self.volume_embed.bias) + \
            ((self.aug_shift_embed.weight,) if self.aug_shift_embed is not None else ())
        key = (self.gemm_precision,) + tuple((p.data_ptr(), p._version) for p in params)
        c = self.__dict__.get("_packed")
        if c is not None and c[0] == key:
            return c[1]
        w = self.unit_embed.weight.detach().contiguous()
        zero = torch.zeros(256, device=w.device)
        emb = torch.stack([self.f0_embed.weight.detach()[:, 0], self.f0_embed.bias.detach(), zero, zero,
                           self.volume_embed.weight.detach()[:, 0], self.volume_embed.bias.detach(),
                           self.aug_shift_embed.weight.detach()[:, 0] if self.aug_shift_embed is not None else zero])
        P = dict(w=_split(w) if self.gemm_precision == "3xtf32" else w, b=self.unit_embed.bias.detach().contiguous(),
                 emb=emb.contiguous())
        self.__dict__["_packed"] = (key, P)
        return P

    def condition(self, units, f0, volume, spk_id=None, spk_mix_dict=None, aug_shift=None):
        """units [B, n_frames, n_unit], f0 / volume [B, n_frames, 1] -> the decoder's condition [B, n_frames, 256]
        (diffusion/vocoder.py:206-215)"""
        _need_cuda_f32("units", units)
        B, T, _ = units.shape
        with torch.no_grad(), _Gemm(self.gemm_precision) as g:
            P = self._pack()
            x = g.linear(units.reshape(B * T, -1).contiguous(), P["w"], P["b"]).contiguous()
            spk, spk_rows = None, 1
            if self.n_spk is not None and self.n_spk > 1:
                if spk_mix_dict is not None:
                    spk = sum(float(v) * self.spk_embed.weight[int(k) - 1] for k, v in spk_mix_dict.items())
                    spk = spk.reshape(1, 256).contiguous()
                else:
                    spk = self.spk_embed(spk_id.reshape(-1) - 1).reshape(-1, 256).contiguous()
                    spk_rows = spk.shape[0]
                    if spk_rows not in (1, B):
                        raise ValueError("spk_id must hold one id per utterance")
            aug = None
            if self.aug_shift_embed is not None and aug_shift is not None:
                aug = aug_shift.to(torch.float32).reshape(-1).expand(B).contiguous()
            f0c, voc = (t.to(torch.float32).reshape(B, T).contiguous() for t in (f0, volume))
            _k(_lib.lib().b2d_u2c_embed(x.data_ptr(), f0c.data_ptr(), 0, voc.data_ptr(), P["emb"].data_ptr(),
                                        0 if spk is None else spk.data_ptr(), spk_rows,
                                        0 if aug is None else aug.data_ptr(), B, T, _stream()), "b2d_u2c_embed")
        return x.reshape(B, T, 256)

    def forward(self, units, f0, volume, spk_id=None, spk_mix_dict=None, aug_shift=None, vocoder=None, gt_spec=None,
                infer=True, infer_speedup=10, method='dpm-solver', k_step=300, use_tqdm=True, noise=None,
                step_noise=None):
        """-> the mel [B, n_frames, M] (diffusion/vocoder.py:196-218)"""
        if not infer:
            raise NotImplementedError(_TRAINING % ("Unit2Mel", "Unit2Mel"))
        x = self.condition(units, f0, volume, spk_id=spk_id, spk_mix_dict=spk_mix_dict, aug_shift=aug_shift)
        x = self.decoder(x, gt_spec=gt_spec, infer=infer, infer_speedup=infer_speedup, method=method, k_step=k_step,
                         use_tqdm=use_tqdm, noise=noise, step_noise=step_noise)
        return x


def _cascade(self, cond_of, units, f0, volume, spk_id, spk_mix_dict, aug_shift, vocoder, gt_spec, infer, return_wav,
             infer_speedup, method, k_step, use_tqdm, ddsp_noise, noise, step_noise, rand_ini, sine_noise):
    """Unit2Wav.forward / Unit2WavFast.forward (diffusion/vocoder.py:237-266, :285-314); ``cond_of(hidden, ddsp_mel)``
    picks the sampler's condition"""
    if not infer:
        raise NotImplementedError(_TRAINING % (type(self).__name__, type(self).__name__))
    ddsp_wav, hidden, (_, _) = self.ddsp_model(units, f0, volume, spk_id=spk_id, spk_mix_dict=spk_mix_dict,
                                               aug_shift=aug_shift, infer=infer, noise=ddsp_noise)
    if vocoder is not None:
        ddsp_mel = vocoder.extract(ddsp_wav)
    else:
        ddsp_mel = None
    if gt_spec is not None and ddsp_mel is None:
        ddsp_mel = gt_spec
    if k_step > 0:
        mel = self.diff_model(cond_of(hidden, ddsp_mel), gt_spec=ddsp_mel, infer=True, infer_speedup=infer_speedup,
                              method=method, k_step=k_step, use_tqdm=use_tqdm, noise=noise, step_noise=step_noise)
    else:
        mel = ddsp_mel
    if return_wav:
        return vocoder.infer(mel, f0, rand_ini=rand_ini, noise=sine_noise)
    return mel


class Unit2Wav(nn.Module):
    def __init__(self, sampling_rate, block_size, n_unit, n_spk, use_pitch_aug=False, out_dims=128, n_layers=20,
                 n_chans=512, pcmer_norm=False):
        super().__init__()
        self.ddsp_model = CombSubFast(sampling_rate, block_size, n_unit, n_spk, use_pitch_aug, pcmer_norm=pcmer_norm)
        self.diff_model = GaussianDiffusion(WaveNet(out_dims, n_layers, n_chans, 256), out_dims=out_dims)

    def forward(self, units, f0, volume, spk_id=None, spk_mix_dict=None, aug_shift=None, vocoder=None, gt_spec=None,
                infer=True, return_wav=False, infer_speedup=10, method='dpm-solver', k_step=None, use_tqdm=True,
                ddsp_noise=None, noise=None, step_noise=None, rand_ini=None, sine_noise=None):
        """-> the mel [B, n_frames, M], or with ``return_wav`` the vocoder's audio; the sampler is conditioned on
        CombSubFast's hidden state and skipped for k_step 0"""
        return _cascade(self, lambda hidden, ddsp_mel: hidden, units, f0, volume, spk_id, spk_mix_dict, aug_shift,
                        vocoder, gt_spec, infer, return_wav, infer_speedup, method, k_step, use_tqdm, ddsp_noise, noise,
                        step_noise, rand_ini, sine_noise)


class Unit2WavFast(nn.Module):
    def __init__(self, sampling_rate, block_size, win_length, n_unit, n_spk, use_pitch_aug=False, out_dims=128,
                 n_layers=6, n_chans=512):
        super().__init__()
        self.ddsp_model = CombSubSuperFast(sampling_rate, block_size, win_length, n_unit, n_spk, use_pitch_aug)
        self.diff_model = GaussianDiffusion(NaiveV2Diff(mel_channels=out_dims, dim=n_chans, num_layers=n_layers,
                                                        condition_dim=out_dims, use_mlp=False), out_dims=out_dims)

    def forward(self, units, f0, volume, spk_id=None, spk_mix_dict=None, aug_shift=None, vocoder=None, gt_spec=None,
                infer=True, return_wav=False, infer_speedup=10, method='dpm-solver', k_step=None, use_tqdm=True,
                ddsp_noise=None, noise=None, step_noise=None, rand_ini=None, sine_noise=None):
        """-> the mel [B, n_frames, M], or with ``return_wav`` the vocoder's audio; the sampler is conditioned on the
        mel of CombSubSuperFast's output and skipped for k_step 0"""
        return _cascade(self, lambda hidden, ddsp_mel: ddsp_mel, units, f0, volume, spk_id, spk_mix_dict, aug_shift,
                        vocoder, gt_spec, infer, return_wav, infer_speedup, method, k_step, use_tqdm, ddsp_noise, noise,
                        step_noise, rand_ini, sine_noise)


#: the data fields a DDSP checkpoint must share with the diffusion model to feed its shallow diffusion, in
#: main_diff.py's check_args order
DATA_FIELDS = ("sampling_rate", "block_size", "encoder")


def data_mismatches(ddsp_args, diff_args):
    """the DATA_FIELDS in which the two configs differ, in that order (empty when the DDSP model can feed the diffusion
    model): the comparison of main_diff.py's / batch_infer.py's check_args and infer_gt_mel.py's"""
    return [f for f in DATA_FIELDS if getattr(ddsp_args.data, f) != getattr(diff_args.data, f)]


class DiffGtMel:
    """diffusion/infer_gt_mel.py on the package's cascade.  Beyond the reference, ``__call__`` and ``infer`` take the
    draws (``ddsp_noise`` for Unit2Wav / Unit2WavFast's synthesizer, ``noise``, ``step_noise``, ``rand_ini``,
    ``sine_noise``); absent, each is drawn as without them."""

    def __init__(self, project_path=None, device=None):
        self.project_path = project_path
        self.device = device if device is not None else "cuda"
        self.model = None
        self.vocoder = None
        self.args = None

    def flush_model(self, project_path, ddsp_config=None):
        if (self.model is None) or (project_path != self.project_path):
            model, vocoder, args = load_model_vocoder(project_path, device=self.device)
            if ddsp_config is None or self.check_args(ddsp_config, args):
                self.model = model
                self.vocoder = vocoder
                self.args = args
                self.project_path = project_path

    def check_args(self, args1, args2):
        bad = data_mismatches(args1, args2)
        for field in ("block_size", "sampling_rate", "encoder"):        # infer_gt_mel.py's order
            if field in bad:
                raise ValueError("the DDSP and diffusion models' %s differ" % field)
        return True

    def __call__(self, audio, f0, hubert, volume, acc=1, spk_id=1, k_step=0, method='pndm', spk_mix_dict=None,
                 start_frame=0, ddsp_noise=None, noise=None, step_noise=None, rand_ini=None, sine_noise=None):
        if audio is None:
            input_mel = None
        else:
            input_mel = self.vocoder.extract(audio, self.args.data.sampling_rate)
        draws = dict(noise=noise, step_noise=step_noise)
        if ddsp_noise is not None:
            draws["ddsp_noise"] = ddsp_noise
        out_mel = self.model(hubert, f0, volume, spk_id=spk_id, spk_mix_dict=spk_mix_dict, vocoder=self.vocoder,
                             gt_spec=input_mel, infer=True, infer_speedup=acc, method=method, k_step=k_step,
                             use_tqdm=False, **draws)
        if start_frame > 0:
            out_mel = out_mel[:, start_frame:, :]
            f0 = f0[:, start_frame:, :]
        output = self.vocoder.infer(out_mel, f0, rand_ini=rand_ini, noise=sine_noise)
        if start_frame > 0:
            output = F.pad(output, (start_frame * self.vocoder.vocoder_hop_size, 0))
        return output

    def start_frame(self, silence_front):
        """the first frame vocoded: int(silence_front * vocoder rate / vocoder hop), infer_gt_mel.py:64"""
        return int(silence_front * self.vocoder.vocoder_sample_rate / self.vocoder.vocoder_hop_size)

    def infer(self, audio, f0, hubert, volume, acc=1, spk_id=1, k_step=0, method='pndm', silence_front=0,
              use_silence=False, spk_mix_dict=None, **draws):
        start_frame = self.start_frame(silence_front)
        if use_silence:
            if audio is not None:
                audio = audio[:, start_frame * self.vocoder.vocoder_hop_size:]
            f0 = f0[:, start_frame:, :]
            hubert = hubert[:, start_frame:, :]
            volume = volume[:, start_frame:, :]
            _start_frame = 0
        else:
            _start_frame = start_frame
        audio = self.__call__(audio, f0, hubert, volume, acc=acc, spk_id=spk_id, k_step=k_step, method=method,
                              spk_mix_dict=spk_mix_dict, start_frame=_start_frame, **draws)
        if use_silence:
            if start_frame > 0:
                audio = F.pad(audio, (start_frame * self.vocoder.vocoder_hop_size, 0))
        return audio
