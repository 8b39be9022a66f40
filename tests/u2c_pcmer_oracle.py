"""Plain-torch restatement of the reference's Unit2Control with the PCmer decoder (ddsp/unit2control.py:26-109 with
PCmer(3 layers, 8 heads, 256), ddsp/pcmer.py) on standard nn layers: the oracle of the PCmer backward.

TEST INFRASTRUCTURE ONLY: differentiable by autograd, usable in float64 (``.double()``), with the reference's state-dict
keys and shapes, so the package's seeded weights load strictly.  It reuses the embedding, convolution stack, final norm
and dense_out of oracle/unit2control.py's NaiveUnit2Control and replaces its decoder.  tests/test_oracle_u2c_pcmer_grad.py
pins its gradients to the reference's own class (tests/golden/u2c_pcmer_grad_*.npz); that makes it the oracle for the
full parameter gradients and the large shapes of tests/test_gpu_u2c_pcmer_backward.py, where the reference does not
exist, and the eager network bench_unit2control_pcmer_grad.py compares against.
"""
import math

import torch
import torch.nn as nn

from oracle.unit2control import NaiveUnit2Control
# ---- the PCmer decoder (ddsp/pcmer.py): performer self-attention + conformer convolution module, no active dropout ----
class _PCmerConvModule(nn.Module):
    """LayerNorm -> pointwise conv (dim -> 4 dim) -> GLU -> zero pad 15 | 15 + depthwise conv k = 31 -> Swish -> pointwise
    conv (2 dim -> dim), on [B, T, dim]; the depthwise Conv1d sits under `net.4.conv` as in the reference"""

    def __init__(self, dim, kernel_size=31):
        super().__init__()
        inner = 2 * dim
        dw = nn.Module()
        dw.conv = nn.Conv1d(inner, inner, kernel_size, groups=inner)
        self.net = nn.Sequential(nn.LayerNorm(dim), nn.Identity(), nn.Conv1d(dim, 2 * inner, 1), nn.Identity(), dw,
                                 nn.Identity(), nn.Conv1d(inner, dim, 1), nn.Identity(), nn.Identity())

    def forward(self, x):
        n = self.net
        x = n[2](n[0](x).transpose(1, 2))
        out, gate = x.chunk(2, dim=1)
        x = n[4].conv(torch.nn.functional.pad(out * gate.sigmoid(), (15, 15)))
        return n[6](x * x.sigmoid()).transpose(1, 2)


class _FastAttention(nn.Module):
    def __init__(self, dim_head, nb_features):
        super().__init__()
        self.register_buffer("projection_matrix", torch.zeros(nb_features, dim_head))

    def features(self, data, is_query, detach_max, eps=1e-4):
        """the softmax-kernel feature map, the reference's op sequence (ddsp/pcmer.py:14-47)"""
        b, h = data.shape[:2]
        normalizer = data.shape[-1] ** -0.25
        ratio = self.projection_matrix.shape[0] ** -0.5
        proj = self.projection_matrix.expand(b, h, *self.projection_matrix.shape).type_as(data)
        dd = torch.einsum("...id,...jd->...ij", normalizer * data, proj)
        diag = ((data ** 2).sum(dim=-1) / 2.0 * (normalizer ** 2)).unsqueeze(dim=-1)
        if is_query:
            m = torch.max(dd, dim=-1, keepdim=True).values
            return ratio * (torch.exp(dd - diag - (m.detach() if detach_max else m)) + eps)
        return ratio * torch.exp(dd - diag + eps)

    def forward(self, q, k, v, pcmer_norm, detach_max):
        if pcmer_norm:
            q = q / (q.norm(dim=-1, keepdim=True) + 1e-8)
            k = k / (k.norm(dim=-1, keepdim=True) + 1e-8)
        q, k = self.features(q, True, detach_max), self.features(k, False, detach_max)
        d_inv = 1. / (torch.einsum("...nd,...d->...n", q, k.sum(dim=-2).type_as(q)) + 1e-8)
        context = torch.einsum("...nd,...ne->...de", k, v)
        return torch.einsum("...de,...nd,...n->...ne", context, q, d_inv)


class _SelfAttention(nn.Module):
    def __init__(self, dim, heads=8, dim_head=64):
        super().__init__()
        self.heads = heads
        self.fast_attention = _FastAttention(dim_head, int(dim_head * math.log(dim_head)))
        self.to_q = nn.Linear(dim, heads * dim_head)
        self.to_k = nn.Linear(dim, heads * dim_head)
        self.to_v = nn.Linear(dim, heads * dim_head)
        self.to_out = nn.Linear(heads * dim_head, dim)

    def forward(self, x, pcmer_norm, detach_max):
        b, n, _ = x.shape
        heads = lambda t: t.reshape(b, n, self.heads, -1).permute(0, 2, 1, 3)            # b n (h d) -> b h n d
        out = self.fast_attention(heads(self.to_q(x)), heads(self.to_k(x)), heads(self.to_v(x)), pcmer_norm, detach_max)
        out = torch.cat([out], dim=1).permute(0, 2, 1, 3)
        return self.to_out(out.reshape(b, n, -1))


class _PCmerLayer(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.conformer = _PCmerConvModule(dim)
        self.norm = nn.LayerNorm(dim)
        self.attn = _SelfAttention(dim)

    def forward(self, x, pcmer_norm, detach_max):
        x = x + self.attn(self.norm(x), pcmer_norm, detach_max)
        return x + self.conformer(x)


class _PCmer(nn.Module):
    def __init__(self, num_layers, dim, owner):
        super().__init__()
        self._layers = nn.ModuleList([_PCmerLayer(dim) for _ in range(num_layers)])
        self.__dict__["owner"] = owner

    def forward(self, x):
        for layer in self._layers:
            x = layer(x, self.owner.pcmer_norm, self.owner.detach_max)
        return x


class PCmerUnit2Control(NaiveUnit2Control):
    """Unit2Control with the PCmer decoder (ddsp/unit2control.py:26-109 with PCmer(3 layers, 8 heads, 256)).  Dropout is
    constructed there but never active (pcmer.py: the layer's residual dropout is never called, attention and convolution
    dropouts are 0), so training mode computes the inference forward.  ``pcmer_norm`` is per instance here (the reference
    keeps it in a process-global flag).  ``detach_max = True`` stops the gradient through the query features' row maximum:
    a wrong variant, for tests that need to show the maximum's term is exercised."""
    detach_max = False

    def __init__(self, input_channel, n_spk, output_splits, use_pitch_aug=False, pcmer_norm=False, use_conv_stack=True):
        super().__init__(input_channel, n_spk, output_splits, use_pitch_aug=use_pitch_aug, use_conv_stack=use_conv_stack)
        self.pcmer_norm = pcmer_norm
        self.decoder = _PCmer(3, 256, self)
