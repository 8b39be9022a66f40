"""Plain-torch restatement of the reflow model's velocity network (reference reflow/naive_v2_diff.py with use_mlp=False,
conv_only=True: what Unit2Wav builds) and of its rectified-flow Euler / RK4 sampler (reflow/reflow.py), on standard nn
layers, usable in float64 (``.double()``), with the reference's state-dict keys and shapes.

TEST INFRASTRUCTURE ONLY.  tests/test_oracle_reflow.py pins it to the reference's own outputs stored by
tests/golden/make_golden_reflow.py; the GPU tests use it (float64 on the CPU, or fp32 eagerly on the GPU: what the
reference runs today) where the reference does not exist.  The convolution module is oracle/unit2control.py's.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.unit2control import _ConvModule


class StepEmbedding(nn.Module):
    """sin / cos of the step times geometric frequencies 10000^(-i / (dim/2 - 1)) in the module's dtype.  The
    frequencies themselves are fp32 in every dtype: the reference computes them from an integer arange, so they are part
    of the model's definition."""

    def __init__(self, dim):
        super().__init__()
        self.dim = dim

    def forward(self, steps, dtype):
        half = self.dim // 2
        freq = torch.exp(torch.arange(half, device=steps.device) * -(math.log(10000) / (half - 1))).to(dtype)
        arg = steps.to(dtype)[:, None] * freq[None, :]
        return torch.cat((arg.sin(), arg.cos()), dim=-1)


class Layer(nn.Module):
    def __init__(self, dim, dim_cond):
        super().__init__()
        self.conformer = _ConvModule(dim)
        self.norm = nn.LayerNorm(dim)                         # in the state dict, unused without attention
        self.diffusion_step_projection = nn.Conv1d(dim, dim, 1)
        self.condition_projection = nn.Conv1d(dim_cond, dim, 1)

    def forward(self, x, cond, step):                         # x [B, dim, T]; the residual is taken before conditioning
        y = x + self.diffusion_step_projection(step) + self.condition_projection(cond)
        return self.conformer(y.transpose(1, 2)).transpose(1, 2) + x


class VelocityNet(nn.Module):
    def __init__(self, mel_channels, dim, condition_dim, num_layers, mlp_factor=4):
        super().__init__()
        self.input_projection = nn.Conv1d(mel_channels, dim, 1)
        self.diffusion_embedding = nn.Sequential(StepEmbedding(dim), nn.Linear(dim, dim * mlp_factor), nn.GELU(),
                                                 nn.Linear(dim * mlp_factor, dim))
        self.residual_layers = nn.ModuleList([Layer(dim, condition_dim) for _ in range(num_layers)])
        self.output_projection = nn.Conv1d(dim, mel_channels, 1)

    def forward(self, spec, diffusion_step, cond):
        """spec [B, 1, M, T] or [B, M, T], diffusion_step [B], cond [B, M_cond, T] -> velocity in spec's layout"""
        four = spec.dim() == 4
        x = spec[:, 0] if four else spec
        dtype = self.input_projection.weight.dtype
        x = F.gelu(self.input_projection(x.to(dtype)))
        e = self.diffusion_embedding[0](diffusion_step, dtype)
        for m in self.diffusion_embedding[1:]:
            e = m(e)
        e = e.unsqueeze(-1)
        cond = cond.to(dtype)
        for layer in self.residual_layers:
            x = layer(x, cond, e)
        v = self.output_projection(x)
        return v[:, None] if four else v


def sample(net, condition, noise, gt_spec=None, infer_step=10, method="euler", t_start=0.0, spec_min=-12, spec_max=2):
    """the rectified-flow sampler in the network's dtype, fed explicit noise [B, 1, M, T]: condition [B, T, M_cond],
    gt_spec [B, T, M] or None -> [B, T, M].  The step times follow the reference's fp32 arithmetic (t += dt)."""
    dtype = net.input_projection.weight.dtype
    cond = condition.to(dtype).transpose(1, 2)
    B = condition.shape[0]
    t_start = max(t_start, 0.0)
    norm = lambda v: (v - spec_min) / (spec_max - spec_min) * 2 - 1
    if gt_spec is None:
        x, t, dt = noise.to(dtype), torch.zeros(B, device=noise.device), 1.0 / infer_step
    else:
        x = t_start * norm(gt_spec.to(dtype)).transpose(1, 2)[:, None] + (1 - t_start) * noise.to(dtype)
        t, dt = torch.full((B,), float(t_start), device=noise.device), (1.0 - t_start) / infer_step
    v = lambda x, s: net(x, 1000 * s, cond)
    for _ in range(infer_step):
        if method == "euler":
            x = x + v(x, t) * dt
        elif method == "rk4":
            k1 = v(x, t)
            k2 = v(x + 0.5 * k1 * dt, t + 0.5 * dt)
            k3 = v(x + 0.5 * k2 * dt, t + 0.5 * dt)
            k4 = v(x + k3 * dt, t + dt)
            x = x + (k1 + 2 * k2 + 2 * k3 + k4) * dt / 6
        else:
            raise NotImplementedError(method)
        t = t + dt
    return (x[:, 0].transpose(1, 2) + 1) / 2 * (spec_max - spec_min) + spec_min


def seeded_weights(net, seed, gain=1.0):
    """every parameter non-zero: weights N(0, gain^2 / fan_in), biases N(0, 0.1^2), LayerNorm weights 1 + N(0, 0.1^2);
    with gain 1 each layer's residual update is of the order of its input and the velocity of order 1"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in net.named_parameters():
            if name.endswith("bias"):
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
            elif ".norm." in name:
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g))
            else:
                fan_in = p[0].numel()
                p.copy_(gain * torch.randn(p.shape, generator=g) / math.sqrt(fan_in))
            p.masked_fill_(p == 0, 1e-3)                      # fp32 randn does return exact zeros (2 in 1M here)
    return net
