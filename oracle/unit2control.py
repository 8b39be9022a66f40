"""Plain-torch restatement of the reference's Unit2Control with the convolution-only decoder (ddsp/unit2control.py:26-109
with ConformerNaiveEncoder(conv_only=True, conv_dropout=0), diffusion/model_conformer_naive.py) on standard nn layers.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): differentiable by autograd, usable in float64 (``.double()``), with the
reference's state-dict keys and shapes, so the package's seeded weights load strictly.  tests/test_oracle_u2c_grad.py pins
its gradients to the reference's own class (tests/golden/u2c_grad_*.npz); that makes it the oracle for the full parameter
gradients and the large shapes of tests/test_gpu_unit2control_backward.py, where the reference does not exist.
"""
import math

import torch
import torch.nn as nn
from torch.nn.utils import weight_norm


class _ConvModule(nn.Module):
    """pointwise conv (dim -> 4 dim) -> GLU -> depthwise conv k = 31 -> SiLU -> pointwise conv (2 dim -> dim); the
    Identity entries keep the parameter-free slots of the reference's Sequential, hence its indices 2, 4, 6"""

    def __init__(self, dim, kernel_size=31):
        super().__init__()
        inner = 2 * dim
        self.net = nn.Sequential(nn.Identity(), nn.Identity(), nn.Conv1d(dim, 2 * inner, 1), nn.GLU(dim=1),
                                 nn.Conv1d(inner, inner, kernel_size, padding=kernel_size // 2, groups=inner), nn.SiLU(),
                                 nn.Conv1d(inner, dim, 1), nn.Identity(), nn.Identity())

    def forward(self, x):                                     # [B, T, dim]
        return self.net(x.transpose(1, 2)).transpose(1, 2)


class _Layer(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.conformer = _ConvModule(dim)
        self.norm = nn.LayerNorm(dim)                         # in the state dict, unused without attention

    def forward(self, x):
        return x + self.conformer(x)


class _Encoder(nn.Module):
    def __init__(self, num_layers, dim):
        super().__init__()
        self.encoder_layers = nn.ModuleList([_Layer(dim) for _ in range(num_layers)])

    def forward(self, x):
        for layer in self.encoder_layers:
            x = layer(x)
        return x


class NaiveUnit2Control(nn.Module):
    def __init__(self, input_channel, n_spk, output_splits, use_pitch_aug=False, use_conv_stack=True):
        super().__init__()
        self.output_splits = output_splits
        self.f0_embed = nn.Linear(1, 256)
        self.phase_embed = nn.Linear(1, 256)
        self.volume_embed = nn.Linear(1, 256)
        self.n_spk = n_spk
        if n_spk is not None and n_spk > 1:
            self.spk_embed = nn.Embedding(n_spk, 256)
        self.aug_shift_embed = nn.Linear(1, 256, bias=False) if use_pitch_aug else None
        if use_conv_stack:
            self.stack = nn.Sequential(nn.Conv1d(input_channel, 256, 3, 1, 1), nn.GroupNorm(4, 256), nn.LeakyReLU(),
                                       nn.Conv1d(256, 256, 3, 1, 1))
        else:
            self.stack = nn.Conv1d(input_channel, 256, 3, 1, 1)
        self.decoder = _Encoder(3, 256)
        self.norm = nn.LayerNorm(256)
        self.n_out = sum(output_splits.values())
        self.dense_out = weight_norm(nn.Linear(256, self.n_out))

    def forward(self, units, f0, phase, volume, spk_id=None, spk_mix_dict=None, aug_shift=None):
        """-> (dict of [B, T, feat] views of one dense tensor, hidden [B, T, 256])"""
        x = self.stack(units.transpose(1, 2)).transpose(1, 2)
        x = x + self.f0_embed((1 + f0 / 700).log()) + self.phase_embed(phase / math.pi) + self.volume_embed(volume)
        if self.n_spk is not None and self.n_spk > 1:
            if spk_mix_dict is not None:
                for k, v in spk_mix_dict.items():
                    x = x + v * self.spk_embed(torch.tensor([[int(k) - 1]], device=units.device))
            else:
                x = x + self.spk_embed(spk_id - 1)
        if self.aug_shift_embed is not None and aug_shift is not None:
            x = x + self.aug_shift_embed(aug_shift / 5)
        x = self.norm(self.decoder(x))
        e = self.dense_out(x)
        return dict(zip(self.output_splits, torch.split(e, list(self.output_splits.values()), dim=-1))), x
