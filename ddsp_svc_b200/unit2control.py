"""Unit2Control inference on the GPU (SURVEY 8f rank 1): the control network that sits between the phase scan and the
synthesis kernels on every call -- reference ddsp/unit2control.py:26-109 with its two decoders, PCmer (performer
attention + conformer convolution, ddsp/pcmer.py) and the convolution-only ConformerNaiveEncoder
(diffusion/model_conformer_naive.py, what configs/combsub.yaml selects).

Same constructor, same parameter tree (state-dict keys and shapes: a checkpoint of the reference loads strictly) and the
same ``forward(units, f0, phase, volume, spk_id=, spk_mix_dict=, aug_shift=) -> (controls dict, hidden)`` contract: the
controls are strided views of ONE dense [B, T, n_out] tensor, which is what the synthesis kernels consume without a copy.

Execution: activations stay token-major [B, T, C].  Plain GEMMs (the k = 3 convolutions as one product over the three
shifted inputs, 1 x 1 convolutions, attention projections and contractions, dense_out) are library GEMMs (cuBLAS through
torch.addmm / bmm, fp32); everything between them runs in the fused kernels of csrc/unit2control.cu (embedding sum,
GroupNorm + LeakyReLU, LayerNorm, GLU + depthwise k = 31 convolution + SiLU, performer feature maps).  Inference only
(the reference's train.py keeps using its own class); CPU tensors raise.
"""
import math

import numpy as np
import torch
import torch.nn as nn
from torch.nn.utils import weight_norm

from . import _lib
from .ops import _count, _need_cuda_f32, _stream


def split_to_dict(tensor, tensor_splits):
    """Split the last dimension into a dict of views (reference ddsp/unit2control.py:12-23)."""
    labels, sizes = list(tensor_splits.keys()), list(tensor_splits.values())
    return dict(zip(labels, torch.split(tensor, sizes, dim=-1)))


class _Noop(nn.Module):
    """parameter-free place holder that keeps the reference's Sequential indices (Transpose, GLU, Swish, Dropout, ...)"""

    def forward(self, x):
        return x


class _DepthWise(nn.Module):                     # ddsp/pcmer.py:177-185 keeps its Conv1d under `.conv`
    def __init__(self, chan, kernel_size):
        super().__init__()
        self.conv = nn.Conv1d(chan, chan, kernel_size, groups=chan)


class _ConvModule(nn.Module):
    """Parameter container of ConformerConvModule (pcmer.py:187-216 with LayerNorm at index 0 and `4.conv`;
    model_conformer_naive.py:113-150 with Identity at index 0 and a plain depthwise Conv1d at index 4)."""

    def __init__(self, dim, naive, expansion_factor=2, kernel_size=31):
        super().__init__()
        inner = dim * expansion_factor
        self.naive = naive
        dw = nn.Conv1d(inner, inner, kernel_size, padding=kernel_size // 2, groups=inner) if naive else _DepthWise(inner, kernel_size)
        self.net = nn.Sequential(_Noop() if naive else nn.LayerNorm(dim), _Noop(), nn.Conv1d(dim, inner * 2, 1), _Noop(), dw,
                                 _Noop(), nn.Conv1d(inner, dim, 1), _Noop(), _Noop())

    def dw_conv(self):
        return self.net[4] if self.naive else self.net[4].conv


def _orthogonal_features(nb_rows, nb_columns):
    """Random orthogonal feature matrix of the performer (pcmer.py:231-259): only the INITIAL value -- checkpoints carry
    the matrix as a buffer."""
    blocks = []
    for _ in range(math.ceil(nb_rows / nb_columns)):
        q, _ = torch.linalg.qr(torch.randn(nb_columns, nb_columns), mode="reduced")
        blocks.append(q.t())
    final = torch.cat(blocks)[:nb_rows]
    return torch.diag(torch.randn(nb_rows, nb_columns).norm(dim=1)) @ final


class _FastAttention(nn.Module):
    def __init__(self, dim_heads):
        super().__init__()
        self.register_buffer("projection_matrix", _orthogonal_features(int(dim_heads * math.log(dim_heads)), dim_heads))


class _SelfAttention(nn.Module):                 # pcmer.py:311-381: heads = 8, dim_head = 64 -> inner 512
    def __init__(self, dim, heads=8, dim_head=64):
        super().__init__()
        self.heads, self.dim_head = heads, dim_head
        self.fast_attention = _FastAttention(dim_head)
        self.to_q = nn.Linear(dim, heads * dim_head)
        self.to_k = nn.Linear(dim, heads * dim_head)
        self.to_v = nn.Linear(dim, heads * dim_head)
        self.to_out = nn.Linear(heads * dim_head, dim)


class _PCmerLayer(nn.Module):                    # pcmer.py:118-156
    def __init__(self, dim, heads):
        super().__init__()
        self.conformer = _ConvModule(dim, naive=False)
        self.norm = nn.LayerNorm(dim)
        self.attn = _SelfAttention(dim, heads)


class _NaiveLayer(nn.Module):                    # model_conformer_naive.py:60-110 with conv_only=True
    def __init__(self, dim):
        super().__init__()
        self.conformer = _ConvModule(dim, naive=True)
        self.norm = nn.LayerNorm(dim)            # present in the reference's state dict, unused when conv_only


class _PCmer(nn.Module):
    def __init__(self, num_layers, heads, dim):
        super().__init__()
        self._layers = nn.ModuleList([_PCmerLayer(dim, heads) for _ in range(num_layers)])


class _NaiveEncoder(nn.Module):
    def __init__(self, num_layers, dim):
        super().__init__()
        self.encoder_layers = nn.ModuleList([_NaiveLayer(dim) for _ in range(num_layers)])


def _k(lib_call, what):
    _lib.check(lib_call, what)
    _count(1)


def _split(x):
    """x -> (hi, lo): TF32-exact parts with hi + lo = x to 2^-22 (csrc/unit2control.cu, b2d_split_tf32)."""
    x = x.contiguous()
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    _k(_lib.lib().b2d_split_tf32(x.data_ptr(), hi.data_ptr(), lo.data_ptr(), x.numel(), _stream()), "b2d_split_tf32")
    return hi, lo


class _Gemm:
    """The library GEMMs of the control network at one of three precisions.

    * ``"3xtf32"`` (default): every product runs as THREE tensor-core GEMMs on TF32-exact operand halves, a_hi b_hi +
      a_lo b_hi + a_hi b_lo with fp32 accumulation -- near-fp32 results at tensor-core speed (against float64: up to
      2.2e-6 relative RMS on the controls, the SIMT fp32 GEMMs 4.6e-7; the tensor cores' accumulators truncate; measured
      on an H100 SXM at 700 W); the halves come from b2d_split_tf32 (weights: once per checkpoint).
    * ``"fp32"``: cuBLAS SIMT fp32 GEMMs (what the reference's Linear layers run on a GPU).
    * ``"tf32"``: one TF32 pass (1e-3 relative per product, under 4e-4 relative RMS on the controls: 3.0e-4 to 3.4e-4
      measured on an H100 SXM at 700 W; the reference's cuDNN convolutions do this under torch's defaults and land at
      1.4e-4).  A single token (B T = 1) runs as matrix-vector products without TF32.
    The TF32 modes flip torch.backends.cuda.matmul.allow_tf32 around their own calls only."""

    def __init__(self, mode):
        if mode not in ("3xtf32", "fp32", "tf32"):
            raise ValueError("gemm_precision must be '3xtf32', 'fp32' or 'tf32'")
        self.mode = mode

    def __enter__(self):
        self.prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = self.mode != "fp32"
        return self

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.allow_tf32 = self.prev
        return False

    def linear(self, x2d, w, bias):
        """x2d [N, K] @ w^T + bias; ``w`` is a packed weight: [O, K] tensor, or (hi, lo) pair in 3xtf32 mode."""
        if self.mode != "3xtf32":
            return torch.addmm(bias, x2d, w.t())
        xh, xl = _split(x2d)
        wh, wl = w
        out = torch.addmm(bias, xh, wh.t())
        out.addmm_(xl, wh.t())
        out.addmm_(xh, wl.t())
        return out

    def matmul(self, a, b):
        """batched a @ b of two activations (the per-head contractions of the linear attention: 256 small problems).
        In 3xtf32 mode these stay fp32 SIMT: cuBLAS serves batched TF32 problems of this shape with sm_80 kernels that are
        slower than its fp32 path here (measured), and splitting both activations costs two more passes."""
        if self.mode != "3xtf32":
            return torch.matmul(a, b)
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            return torch.matmul(a, b)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = True


class Unit2Control(nn.Module):
    #: precision of the library GEMMs, see _Gemm: "3xtf32" (default, fp32-grade on the tensor cores), "fp32", "tf32"
    gemm_precision = "3xtf32"
    #: PCmer: run the performer's linear attention (k-sum, context, normalised read-out) as ONE kernel per (utterance, head)
    #: (csrc/linear_attention.cu) instead of two batched library GEMMs + eager elementwise passes.  Off by default: correct
    #: (same 1.4e-6 on the controls); 256 CTAs of 9 warps, two per SM, single-buffered tiles -- it needs a split over frames
    #: and double buffering to compete with the batched SIMT GEMMs.
    fused_attention = False

    def __init__(self, input_channel, n_spk, output_splits, use_pitch_aug=False, pcmer_norm=False, use_naive_v2=False,
                 use_conv_stack=True):
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
        self.use_conv_stack, self.use_naive_v2, self.pcmer_norm = use_conv_stack, use_naive_v2, pcmer_norm
        self.decoder = _NaiveEncoder(3, 256) if use_naive_v2 else _PCmer(3, 8, 256)
        self.norm = nn.LayerNorm(256)
        self.n_out = sum(output_splits.values())
        self.dense_out = weight_norm(nn.Linear(256, self.n_out))
        self.__dict__["_packed"] = None

    # ---- weights in the layouts the GEMMs / kernels want, rebuilt when a parameter changes (load_state_dict, .to) ----
    def _pack(self):
        key = (self.gemm_precision,) + tuple((p.data_ptr(), p._version) for p in self.parameters()) + \
            tuple((b.data_ptr(), b._version) for b in self.buffers())
        c = self.__dict__.get("_packed")
        if c is not None and c[0] == key:
            return c[1]
        P = {}
        k3 = lambda conv: conv.weight.detach().permute(0, 2, 1).reshape(conv.out_channels, -1).contiguous()   # [O, 3 I]: taps t-1, t, t+1
        if self.use_conv_stack:
            P["c1_w"], P["c1_b"] = k3(self.stack[0]), self.stack[0].bias.detach()
            P["gn_w"], P["gn_b"] = self.stack[1].weight.detach().contiguous(), self.stack[1].bias.detach().contiguous()
            P["c2_w"], P["c2_b"] = k3(self.stack[3]), self.stack[3].bias.detach()
        else:
            P["c1_w"], P["c1_b"] = k3(self.stack), self.stack.bias.detach()
        zero = torch.zeros(256, device=self.f0_embed.weight.device)
        P["emb"] = torch.stack([self.f0_embed.weight.detach()[:, 0], self.f0_embed.bias.detach(),
                                self.phase_embed.weight.detach()[:, 0], self.phase_embed.bias.detach(),
                                self.volume_embed.weight.detach()[:, 0], self.volume_embed.bias.detach(),
                                self.aug_shift_embed.weight.detach()[:, 0] if self.aug_shift_embed is not None else zero]).contiguous()
        layers = []
        for layer in (self.decoder.encoder_layers if self.use_naive_v2 else self.decoder._layers):
            net, L = layer.conformer.net, {}
            if not self.use_naive_v2:
                a = layer.attn
                L["ln_w"], L["ln_b"] = layer.norm.weight.detach().contiguous(), layer.norm.bias.detach().contiguous()
                L["qkv_w"] = torch.cat([a.to_q.weight, a.to_k.weight, a.to_v.weight]).detach().contiguous()
                L["qkv_b"] = torch.cat([a.to_q.bias, a.to_k.bias, a.to_v.bias]).detach().contiguous()
                # feature projection with the d^-1/4 data normaliser folded in (pcmer.py:18,30): [64, 266]
                L["proj_t"] = (a.fast_attention.projection_matrix.detach() * (a.dim_head ** -0.25)).t().contiguous()
                L["out_w"], L["out_b"] = a.to_out.weight.detach(), a.to_out.bias.detach()
                L["cln_w"], L["cln_b"] = net[0].weight.detach().contiguous(), net[0].bias.detach().contiguous()
            dw = layer.conformer.dw_conv()
            L["pw1_w"], L["pw1_b"] = net[2].weight.detach()[:, :, 0].contiguous(), net[2].bias.detach()
            L["dw_w"], L["dw_b"] = dw.weight.detach()[:, 0, :].contiguous(), dw.bias.detach().contiguous()
            L["pw2_w"], L["pw2_b"] = net[6].weight.detach()[:, :, 0].contiguous(), net[6].bias.detach()
            layers.append(L)
        P["layers"] = layers
        P["n_w"], P["n_b"] = self.norm.weight.detach().contiguous(), self.norm.bias.detach().contiguous()
        # weight_norm (old style): w = g v / |v| per output row.  `.weight` itself is only refreshed by the module's forward
        # pre-hook (which never runs here), so it is recomputed from weight_g / weight_v
        P["do_w"] = torch._weight_norm(self.dense_out.weight_v.detach(), self.dense_out.weight_g.detach(), 0).contiguous()
        P["do_b"] = self.dense_out.bias.detach()
        if self.gemm_precision == "3xtf32":          # weights of every GEMM as TF32-exact (hi, lo) pairs, once per checkpoint
            for d in [P] + layers:
                for name in [n for n in d if n.endswith("_w") and n[:-2] in ("c1", "c2", "qkv", "out", "pw1", "pw2", "do")]:
                    d[name] = _split(d[name].contiguous())
                if "proj_t" in d:
                    d["proj"] = _split(d["proj_t"].t().contiguous())        # [J, d] like a Linear weight
        self.__dict__["_packed"] = (key, P)
        return P

    # ---- building blocks ----
    @staticmethod
    def _conv3(g, x, w, b):
        """Conv1d(k = 3, padding 1) on token-major x [B, T, I] as ONE GEMM over the three shifted inputs."""
        xp = torch.nn.functional.pad(x, (0, 0, 1, 1))
        T = x.shape[1]
        cat = torch.cat((xp[:, 0:T], xp[:, 1:T + 1], xp[:, 2:T + 2]), dim=-1)
        return g.linear(cat.reshape(-1, cat.shape[-1]), w, b).reshape(x.shape[0], T, -1)

    @staticmethod
    def _layernorm(x, w, b):
        y = torch.empty_like(x)
        _k(_lib.lib().b2d_u2c_layernorm(x.data_ptr(), y.data_ptr(), x.numel() // x.shape[-1], x.shape[-1], w.data_ptr(),
                                        b.data_ptr(), 1e-5, _stream()), "b2d_u2c_layernorm")
        return y

    def _conv_module(self, g_, x, L, pre_norm):
        B, T, C = x.shape
        h = self._layernorm(x, L["cln_w"], L["cln_b"]) if pre_norm else x
        h = g_.linear(h.reshape(-1, C), L["pw1_w"], L["pw1_b"])                              # [B T, 4 C]: value | gate
        inner = L["dw_w"].shape[0]
        g = torch.empty(B, T, inner, dtype=torch.float32, device=x.device)
        _k(_lib.lib().b2d_u2c_glu_dwconv_silu(h.data_ptr(), L["dw_w"].data_ptr(), L["dw_b"].data_ptr(), g.data_ptr(), B, T, inner,
                                              L["dw_w"].shape[1], _stream()), "b2d_u2c_glu_dwconv_silu")
        return g_.linear(g.reshape(-1, inner), L["pw2_w"], L["pw2_b"]).reshape(B, T, C)

    def _attention(self, g_, x, L):
        """performer self-attention of one PCmer layer on LayerNorm(x) (pcmer.py:148, :220-229, :283-309, :343-381)"""
        B, T, C = x.shape
        a = self.decoder._layers[0].attn
        H, d = a.heads, a.dim_head
        h = self._layernorm(x, L["ln_w"], L["ln_b"])
        qkv = g_.linear(h.reshape(-1, C), L["qkv_w"], L["qkv_b"]).reshape(B, T, 3, H, d)
        q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3).contiguous() for i in range(3))        # [B, H, T, d]
        if self.pcmer_norm:
            q = q / (q.norm(dim=-1, keepdim=True) + 1e-8)
            k = k / (k.norm(dim=-1, keepdim=True) + 1e-8)
        J = L["proj_t"].shape[1]
        feats = []
        zero_bias = torch.zeros(J, device=x.device)
        for data, is_q in ((q, 1), (k, 0)):
            dd = g_.linear(data.reshape(-1, d), L["proj"] if g_.mode == "3xtf32" else L["proj_t"].t(), zero_bias)   # [B H T, J]
            _k(_lib.lib().b2d_u2c_softmax_features(dd.data_ptr(), data.data_ptr(), dd.shape[0], J, d, is_q, 1e-4, _stream()),
               "b2d_u2c_softmax_features")
            feats.append(dd.reshape(B, H, T, J))
        qf, kf = feats
        if self.fused_attention and d == 64 and J <= 272:
            out = torch.empty(B, T, H, d, dtype=torch.float32, device=x.device)
            _k(_lib.lib().b2d_u2c_linear_attention(qf.data_ptr(), kf.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, T, J, d, 1e-8,
                                                   _stream()), "b2d_u2c_linear_attention")
            return g_.linear(out.reshape(B * T, H * d), L["out_w"], L["out_b"]).reshape(B, T, C)
        k_sum = kf.sum(dim=-2)                                                               # [B, H, J]
        d_inv = 1.0 / (torch.einsum("bhnj,bhj->bhn", qf, k_sum) + 1e-8)
        context = g_.matmul(kf.transpose(-1, -2), v)                                         # [B, H, J, d]
        out = g_.matmul(qf, context) * d_inv.unsqueeze(-1)                                   # [B, H, T, d]
        out = out.permute(0, 2, 1, 3).reshape(B * T, H * d)
        return g_.linear(out, L["out_w"], L["out_b"]).reshape(B, T, C)

    @torch.no_grad()
    def forward(self, units, f0, phase, volume, spk_id=None, spk_mix_dict=None, aug_shift=None):
        """units B x n_frames x n_unit; f0, phase, volume B x n_frames x 1 -> (dict of B x n_frames x feat, hidden)"""
        with _Gemm(self.gemm_precision) as g:
            return self._forward(g, units, f0, phase, volume, spk_id, spk_mix_dict, aug_shift)

    def _forward(self, g, units, f0, phase, volume, spk_id=None, spk_mix_dict=None, aug_shift=None):
        _need_cuda_f32("units", units)
        B, T, _ = units.shape
        P = self._pack()
        L = _lib.lib()
        x = self._conv3(g, units, P["c1_w"], P["c1_b"])
        if self.use_conv_stack:
            stats = torch.empty(B * 4 * 2, dtype=torch.float64, device=x.device)
            _k(L.b2d_u2c_groupnorm_lrelu(x.data_ptr(), B, T, 256, 4, P["gn_w"].data_ptr(), P["gn_b"].data_ptr(), 1e-5, 0.01,
                                         stats.data_ptr(), _stream()), "b2d_u2c_groupnorm_lrelu")
            x = self._conv3(g, x, P["c2_w"], P["c2_b"])
        spk, spk_rows = None, 1
        if self.n_spk is not None and self.n_spk > 1:
            if spk_mix_dict is not None:
                spk = sum(float(v) * self.spk_embed.weight[int(k) - 1] for k, v in spk_mix_dict.items()).reshape(1, 256).contiguous()
            else:
                spk = self.spk_embed(spk_id.reshape(-1) - 1).reshape(-1, 256).contiguous()
                spk_rows = spk.shape[0]
                if spk_rows not in (1, B):
                    raise ValueError("spk_id must hold one id per utterance")
        aug = None
        if self.aug_shift_embed is not None and aug_shift is not None:
            aug = aug_shift.to(torch.float32).reshape(-1).expand(B).contiguous()
        f0c, phc, voc = (t.to(torch.float32).reshape(B, T).contiguous() for t in (f0, phase, volume))
        x = x.contiguous()
        _k(L.b2d_u2c_embed(x.data_ptr(), f0c.data_ptr(), phc.data_ptr(), voc.data_ptr(), P["emb"].data_ptr(),
                           0 if spk is None else spk.data_ptr(), spk_rows, 0 if aug is None else aug.data_ptr(), B, T, _stream()),
           "b2d_u2c_embed")
        for Ly in P["layers"]:
            if not self.use_naive_v2:
                x = x + self._attention(g, x, Ly)
            x = x + self._conv_module(g, x, Ly, pre_norm=not self.use_naive_v2)
        x = self._layernorm(x, P["n_w"], P["n_b"])
        e = g.linear(x.reshape(-1, 256), P["do_w"], P["do_b"]).reshape(B, T, self.n_out)
        return split_to_dict(e, self.output_splits), x
