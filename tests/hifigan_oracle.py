"""Plain-torch restatement of the NSF-HiFiGAN generator (reference nsf_hifigan/models.py:207-273, ResBlock1), with the
reference's parameter tree after remove_weight_norm() and the harmonic source given as an input.

TEST INFRASTRUCTURE ONLY.  In float64 (``.double()``) it is the ground truth of the GPU tests; in fp32 under torch's
defaults (cuDNN with TF32) it is what the reference runs today, the eager arm of bench_hifigan.py.
tests/test_oracle_hifigan.py pins it to the reference's own outputs (tests/golden/make_golden_hifigan.py).
"""
import math
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

LRELU_SLOPE = 0.1

# the 44.1 kHz, 128-bin, hop-512 vocoder every config's vocoder.ckpt points at (its config.json)
FULL = dict(resblock="1", num_mels=128, sampling_rate=44100, upsample_rates=[8, 8, 2, 2, 2],
            upsample_kernel_sizes=[16, 16, 4, 4, 4], upsample_initial_channel=512, resblock_kernel_sizes=[3, 7, 11],
            resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]])
# a reduced model with the same hop: three stages of 64 / 32 / 16 channels
SMALL = dict(FULL, upsample_rates=[8, 8, 8], upsample_kernel_sizes=[16, 16, 16], upsample_initial_channel=128)


def config(d):
    """an attribute view of a config dict (the reference's AttrDict is a dict with attribute access)"""
    return SimpleNamespace(**d)


class _Source(nn.Module):
    """only the parameters of SourceModuleHnNSF (the source itself is an input of Generator.forward)"""

    def __init__(self):
        super().__init__()
        self.l_linear = nn.Linear(9, 1)


class ResBlock1(nn.Module):
    def __init__(self, ch, k, dilation):
        super().__init__()
        self.convs1 = nn.ModuleList([nn.Conv1d(ch, ch, k, 1, dilation=d, padding=(k * d - d) // 2) for d in dilation])
        self.convs2 = nn.ModuleList([nn.Conv1d(ch, ch, k, 1, padding=(k - 1) // 2) for _ in dilation])

    def forward(self, x):
        for c1, c2 in zip(self.convs1, self.convs2):
            xt = c2(F.leaky_relu(c1(F.leaky_relu(x, LRELU_SLOPE)), LRELU_SLOPE))
            x = xt + x
        return x


class Generator(nn.Module):
    def __init__(self, h):
        super().__init__()
        self.num_kernels = len(h.resblock_kernel_sizes)
        self.m_source = _Source()
        self.noise_convs = nn.ModuleList()
        c0 = h.upsample_initial_channel
        self.conv_pre = nn.Conv1d(h.num_mels, c0, 7, 1, padding=3)
        self.ups = nn.ModuleList()
        rates = list(h.upsample_rates)
        for i, (u, k) in enumerate(zip(rates, h.upsample_kernel_sizes)):
            c_cur = c0 // (2 ** (i + 1))
            self.ups.append(nn.ConvTranspose1d(c0 // (2 ** i), c_cur, k, u, padding=(k - u) // 2))
            if i + 1 < len(rates):
                s = int(math.prod(rates[i + 1:]))
                self.noise_convs.append(nn.Conv1d(1, c_cur, kernel_size=s * 2, stride=s, padding=s // 2))
            else:
                self.noise_convs.append(nn.Conv1d(1, c_cur, kernel_size=1))
        self.resblocks = nn.ModuleList()
        ch = c0
        for _ in rates:
            ch //= 2
            for k, d in zip(h.resblock_kernel_sizes, h.resblock_dilation_sizes):
                self.resblocks.append(ResBlock1(ch, k, d))
        self.conv_post = nn.Conv1d(ch, 1, 7, 1, padding=3)
        self.upp = int(math.prod(rates))

    def forward(self, x, har):
        """x [B, num_mels, nF], har [B, nF upp, 1] (SourceModuleHnNSF's output) -> [B, 1, nF upp]"""
        dtype = self.conv_pre.weight.dtype
        har = har.to(dtype).transpose(1, 2)
        x = self.conv_pre(x.to(dtype))
        for i, (up, nc) in enumerate(zip(self.ups, self.noise_convs)):
            x = up(F.leaky_relu(x, LRELU_SLOPE)) + nc(har)
            xs = None
            for j in range(self.num_kernels):
                r = self.resblocks[i * self.num_kernels + j](x)
                xs = r if xs is None else xs + r
            x = xs / self.num_kernels
        return torch.tanh(self.conv_post(F.leaky_relu(x)))      # torch's default slope, 0.01 (models.py:260)


def folded_state_dict(sd, dtype=torch.float64):
    """a generator state dict with every weight_g / weight_v pair folded into weight = g v / ||v|| (norm over every dim
    but 0, torch._weight_norm: what remove_weight_norm() computes), in ``dtype``"""
    out = {}
    for k, v in sd.items():
        if k.endswith(".weight_g"):
            continue
        if k.endswith(".weight_v"):
            base = k[:-len("_v")]
            out[base] = torch._weight_norm(v.to(dtype), sd[base + "_g"].to(dtype), 0)
        else:
            out[k] = v.to(dtype)
    return out


def build(h, sd, dtype=torch.float64, fold_dtype=None):
    """the oracle holding the (possibly weight-normed) state dict ``sd``, weight norm folded in ``fold_dtype`` (default
    ``dtype``; torch.float32 is what remove_weight_norm() on an fp32 module does)"""
    net = Generator(h)
    net.load_state_dict(folded_state_dict(sd, fold_dtype or dtype), strict=True)
    return net.to(dtype).eval()


def packed_conv(x, wp, bias, N, k, d):
    """a convolution computed from hifigan.pack_conv's layout the way the kernel reads it, with the weights hi + lo:
    x [B, T, C] float64, wp the packed weights -> [B, T, N] (zero padding at the utterance's edges)"""
    B, T, C = x.shape
    wf = wp.to(torch.float64).reshape(k, C // 8, N // 8, 8, 4, 2, 2)               # [j, kb, nb, g, t, hi|lo, h]
    wf = wf[..., 0, :] + wf[..., 1, :]
    W = wf.permute(2, 3, 1, 5, 4, 0).reshape(N, C, k)                              # n = 8 nb + g, c = 8 kb + 4 h + t
    halo = d * (k - 1) // 2
    xp = F.pad(x.to(torch.float64), (0, 0, halo, halo))
    out = bias.to(torch.float64).expand(B, T, N).clone()
    for j in range(k):
        out += xp[:, j * d:j * d + T] @ W[:, :, j].t()
    return out
