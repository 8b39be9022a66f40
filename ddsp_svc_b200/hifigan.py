"""Drop-in for the NSF-HiFiGAN generator (reference nsf_hifigan/models.py:207-273), inference on the kernels of
csrc/hifigan.cu.

``Generator(h)`` builds the reference's parameter tree: ``conv_pre``, ``ups.i``, ``resblocks.j.convs1/convs2.k`` and
``conv_post`` under ``torch.nn.utils.weight_norm`` (``weight_g`` / ``weight_v`` until ``remove_weight_norm()``),
``noise_convs.i`` plain, ``m_source`` the package's fused SourceModuleHnNSF.  A reference checkpoint's ``generator``
dict loads with ``strict=True`` before and after ``remove_weight_norm()``, so ``nsf_hifigan.models.load_model`` builds
and loads this class unchanged.

The forward runs every convolution as one 3xTF32 tensor-core launch (``ops.hifigan_conv``): ``conv_pre``, each stage's
ConvTranspose1d in polyphase form with its noise_convs term fused, six launches per ResBlock1 whose last one
accumulates the multi-receptive-field sum, and ``ops.hifigan_post``.  The weights are packed once per checkpoint (weight
norm folded, the transposed convolutions in polyphase form, every convolution in the kernel's fragment order) and
re-packed only when a parameter changes, so after the first call a forward reads nothing back from the device.
"""
import math

import torch
import torch.nn as nn
from torch.nn.utils import remove_weight_norm, weight_norm

from . import ops
from .sinegen import SourceModuleHnNSF


def _get(h, name):
    return h[name] if isinstance(h, dict) else getattr(h, name)


def validate(h):
    """raise ValueError naming the field of a configuration the kernels do not implement"""
    if str(_get(h, "resblock")) != "1":
        raise ValueError("resblock: only ResBlock1 ('1') is implemented, got %r" % (_get(h, "resblock"),))
    rates, kernels = list(_get(h, "upsample_rates")), list(_get(h, "upsample_kernel_sizes"))
    if len(rates) != len(kernels) or not rates:
        raise ValueError("upsample_kernel_sizes: one per upsample rate")
    for u, k in zip(rates, kernels):
        if u <= 0 or u % 2:
            raise ValueError("upsample_rates: every rate must be even, got %r" % (rates,))
        if k != 2 * u:
            raise ValueError("upsample_kernel_sizes: each must be twice its rate, got %r for rates %r" % (kernels, rates))
    if _get(h, "num_mels") % 16:
        raise ValueError("num_mels: must be a multiple of 16, got %r" % (_get(h, "num_mels"),))
    c0 = _get(h, "upsample_initial_channel")
    if c0 <= 0 or c0 % (16 << len(rates)):
        raise ValueError("upsample_initial_channel: every stage's channel count (%d halved %d times) must be a multiple "
                         "of 16" % (c0, len(rates)))
    ks, ds = list(_get(h, "resblock_kernel_sizes")), list(_get(h, "resblock_dilation_sizes"))
    if not ks or len(ks) != len(ds):
        raise ValueError("resblock_dilation_sizes: one dilation triple per resblock kernel size")
    for k in ks:
        if k <= 0 or k % 2 == 0:
            raise ValueError("resblock_kernel_sizes: must be odd, got %r" % (ks,))
    for k, d in zip(ks, ds):
        if len(d) != 3 or min(d) <= 0 or max(d) * (k - 1) // 2 > 256:
            raise ValueError("resblock_dilation_sizes: three positive dilations with a halo d (k - 1) / 2 <= 256, "
                             "got %r" % (d,))


def folded_weight(conv):
    """the convolution's weight with weight norm folded, g v / ||v|| (norm over every dim but 0: per output channel of a
    Conv1d, per INPUT channel of a ConvTranspose1d, whose weight is [C_in, C_out, k]), as remove_weight_norm computes it"""
    if hasattr(conv, "weight_g"):
        return torch._weight_norm(conv.weight_v, conv.weight_g, 0)
    return conv.weight


def tf32_round(x):
    """fp32 -> the nearest TF32 value (ties to even), as tf32_rn in csrc/tf32_split.cuh does for finite values"""
    u = x.contiguous().view(torch.int32)
    return ((u + 0xFFF + ((u >> 13) & 1)) & -0x2000).view(torch.float32)


def pack_conv(w):
    """Conv1d weight [N, C_in, k] fp32 -> the kernel's layout [k][C_in / 8][N / 8][32 lanes][4] (flat): lane 4 g + t
    holds the TF32 hi halves of W[8 nb + g, 8 kb + t, j] and W[8 nb + g, 8 kb + t + 4, j], then their lo halves
    (W - hi rounded to TF32)"""
    N, C, k = w.shape
    f = w.reshape(N // 8, 8, C // 8, 2, 4, k).permute(5, 2, 0, 1, 4, 3).reshape(k, C // 8, N // 8, 32, 2)
    hi = tf32_round(f)
    return torch.cat((hi, tf32_round(f - hi)), dim=-1).reshape(-1)


def polyphase(w, u):
    """ConvTranspose1d(C_in, C_out, 2u, stride u, padding u / 2) weight [C_in, C_out, 2u] -> the equivalent k = 3
    Conv1d weight [u C_out, C_in, 3] over input frames m - 1, m, m + 1: output sample m u + r, channel co is column
    r C_out + co, and its tap j (frame m + j - 1) is the original tap r + u / 2 - (j - 1) u, zero outside [0, 2u)"""
    C_in, C_out, K = w.shape
    r = torch.arange(u, device=w.device)[:, None]
    taps = r + u // 2 - (torch.arange(3, device=w.device)[None, :] - 1) * u          # [u, 3]
    valid = (taps >= 0) & (taps < K)
    g = w[:, :, taps.clamp(0, K - 1)] * valid                                         # [C_in, C_out, u, 3]
    return g.permute(2, 1, 0, 3).reshape(u * C_out, C_in, 3)


class ResBlock1(nn.Module):
    """the reference's ResBlock1 parameter tree (models.py:36-76); its forward runs inside Generator.forward"""

    def __init__(self, h, channels, kernel_size=3, dilation=(1, 3, 5)):
        super().__init__()
        self.h = h
        pad = lambda d: (kernel_size * d - d) // 2
        self.convs1 = nn.ModuleList([weight_norm(nn.Conv1d(channels, channels, kernel_size, 1, dilation=d,
                                                           padding=pad(d))) for d in dilation])
        self.convs2 = nn.ModuleList([weight_norm(nn.Conv1d(channels, channels, kernel_size, 1, dilation=1,
                                                           padding=pad(1))) for _ in dilation])

    def remove_weight_norm(self):
        for conv in list(self.convs1) + list(self.convs2):
            remove_weight_norm(conv)


class Generator(nn.Module):
    """Generator(h): the reference's constructor and parameter tree (models.py:207-264); forward(x [B, num_mels, nF]
    (any strides, e.g. NsfHifiGAN's mel.transpose(1, 2)), f0 [B, nF], rand_ini=None, noise=None) -> [B, 1, nF upp].
    rand_ini / noise pass through to m_source (SourceModuleHnNSF.forward), so seeded runs can be compared.  Inference
    only: CUDA fp32 inputs; under grad with trainable parameters in training mode it raises NotImplementedError."""

    def __init__(self, h):
        super().__init__()
        validate(h)
        self.h = h
        self.num_kernels = len(_get(h, "resblock_kernel_sizes"))
        self.num_upsamples = len(_get(h, "upsample_rates"))
        self.m_source = SourceModuleHnNSF(sampling_rate=_get(h, "sampling_rate"), harmonic_num=8)
        self.noise_convs = nn.ModuleList()
        c0 = _get(h, "upsample_initial_channel")
        self.conv_pre = weight_norm(nn.Conv1d(_get(h, "num_mels"), c0, 7, 1, padding=3))
        rates = list(_get(h, "upsample_rates"))
        self.ups = nn.ModuleList()
        for i, (u, k) in enumerate(zip(rates, _get(h, "upsample_kernel_sizes"))):
            c_cur = c0 // (2 ** (i + 1))
            self.ups.append(weight_norm(nn.ConvTranspose1d(c0 // (2 ** i), c_cur, k, u, padding=(k - u) // 2)))
            if i + 1 < len(rates):
                s = int(math.prod(rates[i + 1:]))
                self.noise_convs.append(nn.Conv1d(1, c_cur, kernel_size=s * 2, stride=s, padding=s // 2))
            else:
                self.noise_convs.append(nn.Conv1d(1, c_cur, kernel_size=1))
        self.resblocks = nn.ModuleList()
        ch = c0
        for i in range(len(self.ups)):
            ch //= 2
            for k, d in zip(_get(h, "resblock_kernel_sizes"), _get(h, "resblock_dilation_sizes")):
                self.resblocks.append(ResBlock1(h, ch, k, d))
        self.conv_post = weight_norm(nn.Conv1d(ch, 1, 7, 1, padding=3))
        self.upp = int(math.prod(rates))

    def remove_weight_norm(self):
        for conv in self.ups:
            remove_weight_norm(conv)
        for block in self.resblocks:
            block.remove_weight_norm()
        remove_weight_norm(self.conv_pre)
        remove_weight_norm(self.conv_post)

    # ---- weights in the kernel's layouts, rebuilt when a parameter changes (load_state_dict, .to, remove_weight_norm) ----
    def _pack(self):
        key = tuple((p.data_ptr(), p._version) for p in self.parameters())
        c = self.__dict__.get("_packed")
        if c is not None and c[0] == key:
            return c[1]
        f32 = lambda t: t.detach().float().contiguous()
        conv = lambda m: dict(w=pack_conv(f32(folded_weight(m))), b=f32(m.bias), k=m.kernel_size[0],
                              d=m.dilation[0])
        stages = []
        for i, (up, nc) in enumerate(zip(self.ups, self.noise_convs)):
            u = up.stride[0]
            blocks = [dict(c1=[conv(m) for m in rb.convs1], c2=[conv(m) for m in rb.convs2])
                      for rb in self.resblocks[i * self.num_kernels:(i + 1) * self.num_kernels]]
            stages.append(dict(u=u, c_out=up.out_channels, w=pack_conv(polyphase(f32(folded_weight(up)), u)),
                               b=f32(up.bias), nw=f32(nc.weight).reshape(nc.out_channels, -1), nb=f32(nc.bias),
                               ns=nc.stride[0], npad=nc.padding[0], blocks=blocks))
        post = f32(folded_weight(self.conv_post))[0].t().contiguous()          # [7, C]
        P = dict(pre=conv(self.conv_pre), stages=stages, post_w=post, post_b=f32(self.conv_post.bias))
        self.__dict__["_packed"] = (key, P)
        return P

    def forward(self, x, f0, rand_ini=None, noise=None):
        if not (isinstance(x, torch.Tensor) and x.is_cuda and isinstance(f0, torch.Tensor) and f0.is_cuda):
            raise ValueError("Generator runs on the CUDA kernels: x and f0 must be CUDA tensors")
        if torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("the NSF-HiFiGAN generator is inference-only; call it under torch.no_grad() "
                                      "or in eval() mode")
        with torch.no_grad():
            P = self._pack()
            B, _, T = x.shape
            har = self.m_source(f0, self.upp, rand_ini, noise)                  # [B, nF upp, 1]
            pre = P["pre"]
            h = ops.hifigan_conv(x.transpose(1, 2), pre["w"], pre["b"], pre["k"], pre["d"], pre["b"].numel(), False)
            for st in P["stages"]:
                u, C = st["u"], st["c_out"]
                xu = ops.hifigan_conv(h, st["w"], st["b"], 3, 1, u * C, True, up=u, source=har, noise_w=st["nw"],
                                      noise_b=st["nb"], noise_stride=st["ns"], noise_pad=st["npad"])
                T *= u
                t, y, xs = (torch.empty(B, T, C, dtype=torch.float32, device=x.device) for _ in range(3))
                nk = len(st["blocks"])
                for j, blk in enumerate(st["blocks"]):
                    inp = xu
                    for l, (c1, c2) in enumerate(zip(blk["c1"], blk["c2"])):
                        ops.hifigan_conv(inp, c1["w"], c1["b"], c1["k"], c1["d"], C, True, out=t)
                        res = xu if l == 0 else y
                        if l < 2:
                            ops.hifigan_conv(t, c2["w"], c2["b"], c2["k"], 1, C, True, residual=res, out=y)
                        else:       # the MRF sum: xs = r, xs += r, ..., the last one (xs + r) / num_kernels into xu
                            last = j == nk - 1
                            ops.hifigan_conv(t, c2["w"], c2["b"], c2["k"], 1, C, True, residual=res,
                                             accum=xs if j else None, div=float(nk) if last else 1.0,
                                             out=xu if last else xs)
                        inp = y
                h = xu
            return ops.hifigan_post(h, P["post_w"], P["post_b"])
