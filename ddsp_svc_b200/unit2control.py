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
GroupNorm + LeakyReLU, LayerNorm, GLU + depthwise k = 31 convolution + SiLU, performer feature maps).  CPU tensors raise.

Training: with the convolution-only decoder (``use_naive_v2=True``: what CombSubSuperFast builds, so configs/combsub.yaml,
reflow.yaml and diffusion-fast.yaml), and with the PCmer decoder when ``pcmer_backward`` is set (what Sins, CombSub and
CombSubFast build: configs/sins.yaml, combsub-old, diffusion-new.yaml), the module is differentiable with respect to all
of its parameters when grad mode is on and a parameter requires grad: ONE autograd Function (_Unit2ControlFunction)
around the whole network whose forward is the inference forward (same kernels, bit-identical outputs; neither decoder has
an active dropout) plus the saved activations, and whose backward walks the layers in reverse on the kernels of
csrc/unit2control_bwd.cu and csrc/pcmer_bwd.cu and library GEMMs.  The inputs are data: units, f0, phase, volume or
aug_shift that require grad, and spk_mix_dict under grad, raise NotImplementedError.  With ``pcmer_backward`` off (the
default) the PCmer decoder's outputs are detached in every mode.
"""
import math

import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable
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

    def mm(self, xs, w, bias=None):
        """xs [N, K] @ w^T (+ bias) with xs already in operand form (from ``split``, or from a kernel that writes the
        TF32 halves itself); w packed"""
        if self.mode != "3xtf32":
            return torch.mm(xs, w.t()) if bias is None else torch.addmm(bias, xs, w.t())
        (xh, xl), (wh, wl) = xs, w
        out = torch.mm(xh, wh.t()) if bias is None else torch.addmm(bias, xh, wh.t())
        return out.addmm_(xl, wh.t()).addmm_(xh, wl.t())

    def split(self, x2d):
        """an activation prepared for the products below: (hi, lo) in 3xtf32 mode, itself otherwise"""
        return _split(x2d) if self.mode == "3xtf32" else x2d.contiguous()

    def grad_input(self, gy, w, out=None):
        """(out +) gy [N, O] @ w [O, K]: the adjoint of ``linear`` towards its input; gy from ``split``, w packed"""
        if self.mode != "3xtf32":
            return torch.mm(gy, w) if out is None else out.addmm_(gy, w)
        (gh, gl), (wh, wl) = gy, w
        out = torch.mm(gh, wh) if out is None else out.addmm_(gh, wh)
        return out.addmm_(gl, wh).addmm_(gh, wl)

    def grad_weight(self, gy, x):
        """gy^T [O, N] @ x [N, K]: the adjoint of ``linear`` towards its weight; both operands from ``split``"""
        if self.mode != "3xtf32":
            return torch.mm(gy.t(), x)
        (gh, gl), (xh, xl) = gy, x
        return torch.mm(gh.t(), xh).addmm_(gl.t(), xh).addmm_(gh.t(), xl)

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


class _Unit2ControlFunction(torch.autograd.Function):
    """The whole control network (either decoder) as ONE differentiable op:
    (module, parameter names, inputs..., dense_out weight, *parameters) -> (dense [B, T, n_out], hidden [B, T, 256]).

    forward is Unit2Control._forward as it stands (same kernels and launches, so bit-identical to the no_grad call) and
    keeps: the first convolution's output before GroupNorm + the forward's fp64 statistics, the GroupNorm output, per
    decoder layer the convolution module's input and (PCmer) its LayerNorm output [N, 256], the pw1 output [N, 1024] and
    the GLU-conv-SiLU output [N, 512], the final LayerNorm's input and output (N = B T tokens; about 30 MB per layer at
    24 x 172).  A PCmer layer also keeps its attention's input and LayerNorm output, the qkv projection [N, 1536], the
    feature maps' inputs q, k and v [B, H, T, 64], the features phi_q, phi_k [B, H, T, 266] and the read-out [N, 512]
    (about 170 MB per layer at 24 x 172).  backward walks the layers in reverse: the kernels of csrc/unit2control_bwd.cu
    and csrc/pcmer_bwd.cu (no atomics, fixed summation order: bit-identical from run to run) between library GEMMs at the
    module's gemm_precision (dX = gY W on the packed weights, dW = gY^T X with both activations split in 3xtf32 mode; the
    per-head products through _Gemm.matmul, as in the forward).  Everything inside the GLU -> depthwise conv -> SiLU
    stage is recomputed from the saved pw1 output, and the attention's k-sum, context and normaliser from the saved
    features and v, so one backward serves both fused_attention settings.  Either cotangent may be absent.  Not
    differentiable twice."""

    @staticmethod
    def forward(ctx, mod, names, units, f0, phase, volume, spk_id, aug_shift, do_w, *params):
        save = {}
        with _Gemm(mod.gemm_precision) as g:
            e, hidden = mod._forward(g, units, f0, phase, volume, spk_id, None, aug_shift, save=save)
        ctx.mod, ctx.names, ctx.saved, ctx.spk_id = mod, names, save, spk_id
        ctx.save_for_backward(units, hidden)
        ctx.set_materialize_grads(False)
        return e, hidden

    @staticmethod
    @once_differentiable
    def backward(ctx, ge, gh):
        mod, S = ctx.mod, ctx.saved
        units, hidden = ctx.saved_tensors
        P, (B, T, _) = S["P"], units.shape
        N, n_out, inner, dev = B * T, mod.n_out, P["layers"][0]["dw_w"].shape[0], units.device
        L = _lib.lib()
        max_cols = max([n_out, 2 * inner] + [Ly["qkv_b"].shape[0] for Ly in P["layers"] if "qkv_b" in Ly])
        ws_bytes = L.b2d_u2c_backward_workspace_bytes(B, T, inner, max_cols)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        new = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        unk3 = lambda dw: dw.reshape(dw.shape[0], 3, -1).permute(0, 2, 1).contiguous()        # [O, 3 I] -> Conv1d's [O, I, 3]

        def colsum(g2d):
            out = new(g2d.shape[1])
            _k(L.b2d_u2c_colsum(g2d.data_ptr(), N, g2d.shape[1], out.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "b2d_u2c_colsum")
            return out

        G, d_do_w = {}, None
        with _Gemm(mod.gemm_precision) as g:
            # dense_out, then the final LayerNorm (whose output is also `hidden`)
            if ge is not None:
                ge = ge.contiguous().reshape(N, n_out)
                ges = g.split(ge)
                d_do_w = g.grad_weight(ges, g.split(hidden.reshape(N, 256)))
                G["dense_out.bias"] = colsum(ge)
                gy = g.grad_input(ges, P["do_w"])
                if gh is not None:
                    gy += gh.reshape(N, 256)
            else:
                gy = gh.contiguous().reshape(N, 256)

            def layernorm_backward(x, gy, w, name):
                """-> the cotangent of x through LayerNorm(x); gamma / beta gradients into G[name + ".weight" / ".bias"]"""
                gx, dgb = new(N, 256), new(2, 256)
                _k(L.b2d_u2c_layernorm_backward(x.data_ptr(), gy.data_ptr(), w.data_ptr(), 1e-5, N, 256, gx.data_ptr(), dgb.data_ptr(),
                                                ws.data_ptr(), ws_bytes, _stream()), "b2d_u2c_layernorm_backward")
                G[name + ".weight"], G[name + ".bias"] = dgb[0], dgb[1]
                return gx

            def attention_backward(gy, Ly, A, name):
                """performer self-attention y = to_out(read-out(phi_q, phi_k, v)) on a = LN_a(x) with q, k, v = qkv(a):
                gy [N, 256] the cotangent of y -> that of a; parameter gradients into G[name + ...]"""
                qf, kf, v = A["qf"], A["kf"], A["v"]                                          # [B, H, T, J], [B, H, T, 64]
                H, J, d = qf.shape[1], qf.shape[3], v.shape[3]
                R = B * H * T
                gys = g.split(gy)
                G[name + "to_out.weight"] = g.grad_weight(gys, g.split(A["out"].reshape(N, H * d)))
                G[name + "to_out.bias"] = colsum(gy)
                g_out = g.grad_input(gys, Ly["out_w"])                                        # [N, H d] token-major
                # k-sum, normaliser and context recomputed with the forward's own expressions
                k_sum = kf.sum(dim=-2)
                d_inv = 1.0 / (torch.einsum("bhnj,bhj->bhn", qf, k_sum) + 1e-8)
                context = g.matmul(kf.transpose(-1, -2), v)                                   # [B, H, J, d]
                gn = new(B, H, T, d + 1)                                                      # [g_num | g_D]
                _k(L.b2d_u2c_attn_readout_backward(g_out.data_ptr(), A["out"].data_ptr(), d_inv.data_ptr(), B, H, T, d, gn.data_ptr(),
                                                   _stream()), "b2d_u2c_attn_readout_backward")
                gc = g.matmul(qf.transpose(-1, -2), gn)                                       # [B, H, J, d + 1]: [g_ctx | g_ksum]
                g_ctx = gc[..., :d]
                g_qf = g.matmul(gn[..., :d], context.transpose(-1, -2))                       # [B, H, T, J]
                g_kf = g.matmul(v, g_ctx.transpose(-1, -2))
                g_v = g.matmul(kf, g_ctx)                                                     # [B, H, T, d]
                proj = Ly["proj"] if g.mode == "3xtf32" else Ly["proj_t"].t()
                g_data = []
                for gf, feat, data, vec, scal, is_q in ((g_qf, qf, A["q"], k_sum, gn[..., d].contiguous(), 1),
                                                        (g_kf, kf, A["k"], gc[..., d].contiguous(), None, 0)):
                    gd = new(R, d)
                    _k(L.b2d_u2c_softmax_features_backward(gf.data_ptr(), feat.data_ptr(), data.data_ptr(), vec.data_ptr(),
                                                           0 if scal is None else scal.data_ptr(), R, T, J, d, is_q, 1e-4,
                                                           gd.data_ptr(), _stream()), "b2d_u2c_softmax_features_backward")
                    g_data.append(g.grad_input(g.split(gf.reshape(R, J)), proj, out=gd))
                g_qkv = new(N, 3 * H * d)
                _k(L.b2d_u2c_qkv_gather_backward(g_data[0].data_ptr(), g_data[1].data_ptr(), g_v.data_ptr(), A["qkv"].data_ptr(), B, H,
                                                 T, d, int(mod.pcmer_norm), g_qkv.data_ptr(), _stream()), "b2d_u2c_qkv_gather_backward")
                gqs = g.split(g_qkv)
                dw, db = g.grad_weight(gqs, g.split(A["a"].reshape(N, 256))), colsum(g_qkv)
                for j, part in enumerate(("to_q.", "to_k.", "to_v.")):
                    G[name + part + "weight"], G[name + part + "bias"] = dw[j * H * d:(j + 1) * H * d], db[j * H * d:(j + 1) * H * d]
                return g.grad_input(gqs, Ly["qkv_w"])

            gx = layernorm_backward(S["ln_in"], gy, P["n_w"], "norm")
            # decoder layers: x1 = x + attention(LN_a(x)) (PCmer only), x2 = x1 + pw2(glu_dwconv_silu(pw1(LN_c(x1))))
            naive = mod.use_naive_v2
            for i in reversed(range(len(P["layers"]))):
                lpre = ("decoder.encoder_layers.%d." if naive else "decoder._layers.%d.") % i
                (x_in, hn, h, s), Ly, pre = S["layers"][i], P["layers"][i], lpre + "conformer.net."
                gxs = g.split(gx)
                G[pre + "6.weight"] = g.grad_weight(gxs, g.split(s.reshape(N, inner))).unsqueeze(-1)
                G[pre + "6.bias"] = colsum(gx)
                gs = g.grad_input(gxs, Ly["pw2_w"])
                ghh, dwb = new(N, 2 * inner), new(inner, 32)
                _k(L.b2d_u2c_glu_dwconv_silu_backward(h.data_ptr(), Ly["dw_w"].data_ptr(), Ly["dw_b"].data_ptr(), gs.data_ptr(),
                                                      ghh.data_ptr(), dwb.data_ptr(), B, T, inner, Ly["dw_w"].shape[1], ws.data_ptr(),
                                                      ws_bytes, _stream()), "b2d_u2c_glu_dwconv_silu_backward")
                dw = pre + ("4." if naive else "4.conv.")
                G[dw + "weight"], G[dw + "bias"] = dwb[:, :31].unsqueeze(1).contiguous(), dwb[:, 31].contiguous()
                ghs = g.split(ghh)
                G[pre + "2.weight"] = g.grad_weight(ghs, g.split(hn.reshape(N, 256))).unsqueeze(-1)
                G[pre + "2.bias"] = colsum(ghh)
                if naive:
                    gx = g.grad_input(ghs, Ly["pw1_w"], out=gx)                 # + the residual branch
                    continue
                gx = gx + layernorm_backward(x_in, g.grad_input(ghs, Ly["pw1_w"]), Ly["cln_w"], pre + "0")
                A = S["attn"][i]
                gx = gx + layernorm_backward(A["x"], attention_backward(gx, Ly, A, lpre + "attn."), Ly["ln_w"], lpre + "norm")
            # embedding sum: gx passes through to the stack unchanged
            dtable, rowsum, aug = new(7, 256), new(B, 256), S["aug"]
            _k(L.b2d_u2c_embed_backward(gx.data_ptr(), S["f0"].data_ptr(), S["phase"].data_ptr(), S["volume"].data_ptr(),
                                        0 if aug is None else aug.data_ptr(), B, T, dtable.data_ptr(), rowsum.data_ptr(),
                                        ws.data_ptr(), ws_bytes, _stream()), "b2d_u2c_embed_backward")
            for row, name in enumerate(("f0_embed", "phase_embed", "volume_embed")):
                G[name + ".weight"], G[name + ".bias"] = dtable[2 * row].unsqueeze(1), dtable[2 * row + 1]
            if aug is not None:
                G["aug_shift_embed.weight"] = dtable[6].unsqueeze(1)
            if mod.n_spk is not None and mod.n_spk > 1:
                # utterance b adds its row sum into row spk_id[b] - 1: a one-hot product in fp64 (utterance order, no atomics)
                ids = (ctx.spk_id.reshape(1, -1) - 1).expand(1, B)
                onehot = torch.zeros(mod.n_spk, B, dtype=torch.float64, device=dev).scatter_(0, ids, 1.0)
                G["spk_embed.weight"] = (onehot @ rowsum.double()).float()
            # convolution stack: the first convolution's input is data (dW, db only)
            first = "stack."
            if mod.use_conv_stack:
                first, gxs = "stack.0.", g.split(gx)
                G["stack.3.weight"] = unk3(g.grad_weight(gxs, g.split(mod._gather3(S["y1"]).reshape(N, -1))))
                G["stack.3.bias"] = colsum(gx)
                gcat, gy1, gx, dgb = g.grad_input(gxs, P["c2_w"]), new(N, 256), new(N, 256), new(2, 256)
                _k(L.b2d_u2c_conv3_fold(gcat.data_ptr(), B, T, 256, gy1.data_ptr(), _stream()), "b2d_u2c_conv3_fold")
                _k(L.b2d_u2c_groupnorm_lrelu_backward(S["x1"].data_ptr(), S["stats"].data_ptr(), P["gn_w"].data_ptr(),
                                                      P["gn_b"].data_ptr(), 1e-5, 0.01, gy1.data_ptr(), B, T, 256, 4, gx.data_ptr(),
                                                      dgb.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
                   "b2d_u2c_groupnorm_lrelu_backward")
                G["stack.1.weight"], G["stack.1.bias"] = dgb[0], dgb[1]
            G[first + "weight"] = unk3(g.grad_weight(g.split(gx), g.split(mod._gather3(units).reshape(N, -1))))
            G[first + "bias"] = colsum(gx)
        return (None,) * 8 + (d_do_w,) + tuple(G.get(n) for n in ctx.names)


class Unit2Control(nn.Module):
    #: precision of the library GEMMs, see _Gemm: "3xtf32" (default, fp32-grade on the tensor cores), "fp32", "tf32"
    gemm_precision = "3xtf32"
    #: PCmer: run the performer's linear attention (k-sum, context, normalised read-out) as ONE kernel per (utterance, head)
    #: (csrc/linear_attention.cu) instead of two batched library GEMMs + eager elementwise passes.  Off by default: correct
    #: (same 1.4e-6 on the controls); 256 CTAs of 9 warps, two per SM, single-buffered tiles -- it needs a split over frames
    #: and double buffering to compete with the batched SIMT GEMMs.
    fused_attention = False
    #: PCmer: with grad mode on and a parameter that requires grad, make both outputs differentiable with respect to every
    #: parameter (the backward of _Unit2ControlFunction; the forward issues the same kernels with the same results).  Off by
    #: default: the PCmer decoder's outputs have always been detached and a test pins that; turning the default on is a
    #: separate decision.  Set it on the class (``Unit2Control.pcmer_backward = True``) or per instance.
    pcmer_backward = False

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
        cat = Unit2Control._gather3(x)
        return g.linear(cat.reshape(-1, cat.shape[-1]), w, b).reshape(x.shape[0], x.shape[1], -1)

    @staticmethod
    def _gather3(x):
        """[B, T, I] -> [B, T, 3 I]: rows (x[t-1], x[t], x[t+1]) with zero padding"""
        xp = torch.nn.functional.pad(x, (0, 0, 1, 1))
        T = x.shape[1]
        return torch.cat((xp[:, 0:T], xp[:, 1:T + 1], xp[:, 2:T + 2]), dim=-1)

    @staticmethod
    def _layernorm(x, w, b):
        y = torch.empty_like(x)
        _k(_lib.lib().b2d_u2c_layernorm(x.data_ptr(), y.data_ptr(), x.numel() // x.shape[-1], x.shape[-1], w.data_ptr(),
                                        b.data_ptr(), 1e-5, _stream()), "b2d_u2c_layernorm")
        return y

    def _conv_module(self, g_, x, L, pre_norm, save=None):
        B, T, C = x.shape
        hn = self._layernorm(x, L["cln_w"], L["cln_b"]) if pre_norm else x
        h = g_.linear(hn.reshape(-1, C), L["pw1_w"], L["pw1_b"])                             # [B T, 4 C]: value | gate
        inner = L["dw_w"].shape[0]
        g = torch.empty(B, T, inner, dtype=torch.float32, device=x.device)
        _k(_lib.lib().b2d_u2c_glu_dwconv_silu(h.data_ptr(), L["dw_w"].data_ptr(), L["dw_b"].data_ptr(), g.data_ptr(), B, T, inner,
                                              L["dw_w"].shape[1], _stream()), "b2d_u2c_glu_dwconv_silu")
        if save is not None:
            save["layers"].append((x, hn, h, g))
        return g_.linear(g.reshape(-1, inner), L["pw2_w"], L["pw2_b"]).reshape(B, T, C)

    def _attention(self, g_, x, L, save=None):
        """performer self-attention of one PCmer layer on LayerNorm(x) (pcmer.py:148, :220-229, :283-309, :343-381);
        ``save``: a dict whose "attn" list receives what the backward needs"""
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
        else:
            k_sum = kf.sum(dim=-2)                                                           # [B, H, J]
            d_inv = 1.0 / (torch.einsum("bhnj,bhj->bhn", qf, k_sum) + 1e-8)
            context = g_.matmul(kf.transpose(-1, -2), v)                                     # [B, H, J, d]
            out = g_.matmul(qf, context) * d_inv.unsqueeze(-1)                               # [B, H, T, d]
            out = out.permute(0, 2, 1, 3)
        out = out.reshape(B * T, H * d)
        if save is not None:                 # the feature kernel worked in place: qf, kf are the features, q, k their inputs
            save["attn"].append(dict(x=x, a=h, qkv=qkv, q=q, k=k, v=v, qf=qf, kf=kf, out=out))
        return g_.linear(out, L["out_w"], L["out_b"]).reshape(B, T, C)

    def forward(self, units, f0, phase, volume, spk_id=None, spk_mix_dict=None, aug_shift=None):
        """units B x n_frames x n_unit; f0, phase, volume B x n_frames x 1 -> (dict of B x n_frames x feat, hidden).
        Convolution-only decoder, or PCmer decoder with ``pcmer_backward``, grad mode on and a parameter that requires
        grad: both outputs carry the CUDA backward towards every parameter (module docstring); otherwise the outputs are
        detached."""
        if (self.use_naive_v2 or self.pcmer_backward) and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            for name, t in (("units", units), ("f0", f0), ("phase", phase), ("volume", volume), ("aug_shift", aug_shift)):
                if torch.is_tensor(t) and t.requires_grad:
                    raise NotImplementedError("Unit2Control: no gradient with respect to %s (the inputs are data)" % name)
            if spk_mix_dict is not None:
                raise NotImplementedError("Unit2Control: spk_mix_dict is an inference feature; train with spk_id")
            names, params = self._grad_params()
            # weight norm is parameter-side (once per step, not per token): autograd turns dW into d weight_g, d weight_v
            do_w = torch._weight_norm(self.dense_out.weight_v, self.dense_out.weight_g, 0)
            e, hidden = _Unit2ControlFunction.apply(self, names, units, f0, phase, volume, spk_id, aug_shift, do_w, *params)
            return split_to_dict(e, self.output_splits), hidden
        with torch.no_grad(), _Gemm(self.gemm_precision) as g:
            e, hidden = self._forward(g, units, f0, phase, volume, spk_id, spk_mix_dict, aug_shift)
            return split_to_dict(e, self.output_splits), hidden

    def _grad_params(self):
        """(names, tensors) of the parameters the backward produces gradients for, in the order _Unit2ControlFunction
        returns them: all but dense_out.weight_g / weight_v (reached through the weight-norm product) and the
        convolution-only decoder's layer LayerNorms (in the state dict, unused when conv_only); the PCmer layers' norms are
        used and included.  The performer's projection matrix is a buffer."""
        skip = ("dense_out.weight_g", "dense_out.weight_v")
        items = [(n, p) for n, p in self.named_parameters()
                 if n not in skip and not (n.startswith("decoder.encoder_layers.") and ".norm." in n)]
        return tuple(n for n, _ in items), tuple(p for _, p in items)

    def _forward(self, g, units, f0, phase, volume, spk_id=None, spk_mix_dict=None, aug_shift=None, save=None):
        """-> (dense [B, T, n_out], hidden [B, T, 256]); ``save``: a dict that receives what the backward needs"""
        _need_cuda_f32("units", units)
        B, T, _ = units.shape
        P = self._pack()
        L = _lib.lib()
        x = self._conv3(g, units, P["c1_w"], P["c1_b"])
        if self.use_conv_stack:
            stats = torch.empty(B * 4 * 2, dtype=torch.float64, device=x.device)
            if save is not None:
                save["x1"], save["stats"] = x.clone(), stats       # the GroupNorm kernel works in place
            _k(L.b2d_u2c_groupnorm_lrelu(x.data_ptr(), B, T, 256, 4, P["gn_w"].data_ptr(), P["gn_b"].data_ptr(), 1e-5, 0.01,
                                         stats.data_ptr(), _stream()), "b2d_u2c_groupnorm_lrelu")
            if save is not None:
                save["y1"] = x
            x = self._conv3(g, x, P["c2_w"], P["c2_b"])
        spk, spk_rows = None, 1
        if save is not None:
            save["layers"], save["attn"] = [], []
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
                x = x + self._attention(g, x, Ly, save=save)
            x = x + self._conv_module(g, x, Ly, pre_norm=not self.use_naive_v2, save=save)
        if save is not None:
            save.update(P=P, f0=f0c, phase=phc, volume=voc, aug=aug, ln_in=x)
        x = self._layernorm(x, P["n_w"], P["n_b"])
        e = g.linear(x.reshape(-1, 256), P["do_w"], P["do_b"]).reshape(B, T, self.n_out)
        return e, x
