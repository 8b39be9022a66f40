"""Drop-in for the units encoders (reference ddsp/vocoder.py ``Units_Encoder``; ``HubertSoft`` encoder/hubert/model.py;
the fairseq HuBERT-base / ContentVec checkpoints), inference on the kernels of csrc/hubert.cu and the library GEMMs.

``HubertSoft()`` builds bshall's parameter tree (``feature_extractor.conv0..6`` / ``norm0``, ``feature_projection``,
``positional_embedding.conv`` with old-style weight norm over dim 2, ``norm``, ``encoder.layers`` of
``nn.TransformerEncoderLayer`` (post-LN), ``proj``, and the unused ``masked_spec_embed`` / ``label_embedding``), so a
bshall checkpoint loads with ``strict=True``.  ``load_fairseq_hubert(path)`` maps a fairseq HuBERT-base or ContentVec
checkpoint onto the same tree without importing fairseq.  ``Units_Encoder`` is the reference's class:
``patch_reference(units=True)`` rebinds the name in ddsp.vocoder.

The path: resample to 16 kHz (rv_resample with rmvpe.resample_table), the feature convolutions (conv0 and its
GroupNorm in hb_conv0; convolutions 1-6 as library GEMMs on row pairs of the channel-contiguous activations, no
im2col), LayerNorm + the feature projection, the grouped positional convolution (hb_posconv), and the post-LN
transformer layers (QKV, out-proj and FFN as library GEMMs, hb_attention, hb_ln).  Every GEMM runs in 3xTF32.  Weights
are packed once per model, device and layer count (weight norm folded, q/k/v concatenated, TF32 halves: about 0.75 GB
for the published model) and re-packed only when a parameter changes.
"""
import _compat_pickle
import argparse
import collections.abc
import pickle
import re
import threading
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.modules.utils import consume_prefix_in_state_dict_if_present

from . import ops
from .rmvpe import Resampler
from .unit2control import _Gemm, _split

D_MODEL, N_HEADS, D_FFN, N_LAYERS, C_FEAT = 768, 12, 3072, 12, 512
POS_TAPS, POS_GROUPS = 128, 16
UNITS_PAD = (400 - 320) // 2                     # HubertSoft.units' zero pad on each side
CONV_FEATURE_LAYERS = "[(512,10,5)]+[(512,3,2)]*4+[(512,2,2)]*2"
# encoder kind -> (output layer, final_proj applied, batch flattened into one row as the reference's view(1, -1))
KINDS = {"hubertsoft": (12, True, False),
         "hubertbase": (9, True, False), "hubertbase768": (9, False, False), "hubertbase768l12": (12, False, False),
         "contentvec": (9, True, True), "contentvec768": (9, False, True), "contentvec768l12": (12, False, True)}


# ---- the reference's parameter tree (encoder/hubert/model.py); the forward runs in HubertSoft._run ---------------------
class FeatureExtractor(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv0 = nn.Conv1d(1, C_FEAT, 10, 5, bias=False)
        self.norm0 = nn.GroupNorm(C_FEAT, C_FEAT)
        for i in range(1, 7):
            setattr(self, "conv%d" % i, nn.Conv1d(C_FEAT, C_FEAT, 3 if i <= 4 else 2, 2, bias=False))


class FeatureProjection(nn.Module):
    def __init__(self):
        super().__init__()
        self.norm = nn.LayerNorm(C_FEAT)
        self.projection = nn.Linear(C_FEAT, D_MODEL)


class WeightNormConv(nn.Module):
    """the parameters of ``nn.utils.weight_norm(nn.Conv1d(768, 768, 128, padding=64, groups=16), dim=2)``:
    weight = weight_g * weight_v / ||weight_v|| with one norm per tap over all channels"""

    def __init__(self):
        super().__init__()
        conv = nn.Conv1d(D_MODEL, D_MODEL, POS_TAPS, padding=POS_TAPS // 2, groups=POS_GROUPS)
        v = conv.weight.detach()
        self.weight_g = nn.Parameter(v.norm(dim=(0, 1), keepdim=True))
        self.weight_v = nn.Parameter(v.clone())
        self.bias = nn.Parameter(conv.bias.detach().clone())


class PositionalConvEmbedding(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = WeightNormConv()


class TransformerEncoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.layers = nn.ModuleList([nn.TransformerEncoderLayer(D_MODEL, N_HEADS, D_FFN, activation="gelu",
                                                                batch_first=True) for _ in range(N_LAYERS)])
        self.num_layers = N_LAYERS


def fold_weight_norm(g, v):
    """torch._weight_norm(v, g, dim=2) in float64: v scaled by g / ||v|| per tap (norm over dims 0 and 1)"""
    v = v.double()
    return v * (g.double() / v.norm(dim=(0, 1), keepdim=True))


def pack_posconv(w):
    """the folded positional weight [768 out, 48 in, 128] -> [16 groups, 128 taps, 48 in, 48 out] (hb_posconv)"""
    return w.reshape(POS_GROUPS, D_MODEL // POS_GROUPS, D_MODEL // POS_GROUPS, POS_TAPS).permute(0, 3, 2, 1).contiguous()


def pack_strided_conv(w):
    """Conv1d(512, 512, k, stride 2) weight [512, 512, k] -> the row-pair GEMM weights over P[t] = [x[2t] | x[2t + 1]]:
    k = 3: ([w0 | w1] [512, 1024], w2 [512, 512]), out[t] = P[t] [w0 | w1]^T + x[2t + 2] w2^T with x[2t + 2] the first
    half of P[t + 1]; k = 2: ([w0 | w1], None)"""
    w01 = torch.cat([w[:, :, 0], w[:, :, 1]], dim=1)
    return w01.contiguous(), (w[:, :, 2].contiguous() if w.shape[-1] == 3 else None)


def feature_lengths(n, pad=0):
    """frame counts after conv0 .. conv6 of n samples zero-padded by `pad` on each side"""
    L = [(n + 2 * pad - 10) // 5 + 1]
    for k in (3, 3, 3, 3, 2, 2):
        L.append((L[-1] - k) // 2 + 1)
    return L


def align_index(n_frames, ratio, T):
    """Units_Encoder.encode's frame index min(round(ratio * arange(n_frames)), T - 1) with torch's float32 arithmetic:
    the product rounded to float32, then half to even (numpy restatement of what hb_align computes)"""
    idx = np.rint(np.float32(ratio) * np.arange(n_frames, dtype=np.float32)).astype(np.int64)
    return np.minimum(idx, T - 1)


class HubertSoft(nn.Module):
    """HubertSoft(): the reference's constructor and parameter tree (encoder/hubert/model.py).  units(wav [B, 1, N]
    CUDA) -> [B, T, 256]: the 40-sample zero pad on each side, all 12 layers, proj.  encode(wav [B, 1, N], layer=None)
    -> ([B, T, 768] after `layer` layers (all when None), None).  Inference only."""

    def __init__(self, num_label_embeddings=100):
        super().__init__()
        self.feature_extractor = FeatureExtractor()
        self.feature_projection = FeatureProjection()
        self.positional_embedding = PositionalConvEmbedding()
        self.norm = nn.LayerNorm(D_MODEL)
        self.encoder = TransformerEncoder()
        self.proj = nn.Linear(D_MODEL, 256)
        self.masked_spec_embed = nn.Parameter(torch.FloatTensor(D_MODEL).uniform_())
        self.label_embedding = nn.Embedding(num_label_embeddings, 256)
        self._lock = threading.Lock()

    # ---- weights in the kernels' layouts, rebuilt when a parameter changes ----
    def _pack(self, device, n_layers, proj):
        key = (tuple((t.data_ptr(), t._version) for t in self.parameters()), str(device), n_layers, proj)
        with self._lock:
            c = self.__dict__.get("_packed")
            if c is not None and c[0] == key:
                return c[1]
            self.__dict__["_packed"] = None                         # free the old pack before building the new one
            f32 = lambda t: t.detach().to(device=device, dtype=torch.float32).contiguous()
            with torch.no_grad():
                fe, fp = self.feature_extractor, self.feature_projection
                P = dict(conv0=f32(fe.conv0.weight), gn=(f32(fe.norm0.weight), f32(fe.norm0.bias)), convs=[])
                for i in range(1, 7):
                    w01, w2 = pack_strided_conv(f32(getattr(fe, "conv%d" % i).weight))
                    P["convs"].append((_split(w01), _split(w2) if w2 is not None else None))
                P["fp_norm"] = (f32(fp.norm.weight), f32(fp.norm.bias))
                P["fp"] = (_split(f32(fp.projection.weight)), f32(fp.projection.bias))
                pc = self.positional_embedding.conv
                P["pos"] = (f32(pack_posconv(fold_weight_norm(pc.weight_g.detach().cpu(), pc.weight_v.detach().cpu()))),
                            f32(pc.bias))
                P["norm"] = (f32(self.norm.weight), f32(self.norm.bias))
                P["layers"] = []
                for layer in self.encoder.layers[:n_layers]:
                    at = layer.self_attn
                    P["layers"].append(dict(
                        qkv=(_split(f32(at.in_proj_weight)), f32(at.in_proj_bias)),
                        out=(_split(f32(at.out_proj.weight)), f32(at.out_proj.bias)),
                        n1=(f32(layer.norm1.weight), f32(layer.norm1.bias), float(layer.norm1.eps)),
                        fc1=(_split(f32(layer.linear1.weight)), f32(layer.linear1.bias)),
                        fc2=(_split(f32(layer.linear2.weight)), f32(layer.linear2.bias)),
                        n2=(f32(layer.norm2.weight), f32(layer.norm2.bias), float(layer.norm2.eps))))
                P["proj"] = (_split(f32(self.proj.weight)), f32(self.proj.bias)) if proj else None
            self.__dict__["_packed"] = (key, P)
            return P

    def _check(self, wav):
        if not (isinstance(wav, torch.Tensor) and wav.is_cuda):
            raise ValueError("the units encoder runs on the CUDA kernels: wav must be a CUDA tensor")
        if torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("the units encoder is inference-only; call it under torch.no_grad() or in eval() "
                                      "mode")

    def _run(self, wav, pad=0, n_layers=N_LAYERS, proj=False):
        """wav [B, N] CUDA -> [B, T, 768] after n_layers layers ([B, T, proj rows] with proj)"""
        if wav.dim() != 2:
            raise ValueError("wav must be [B, N], got %s" % (tuple(wav.shape),))
        if not 0 <= n_layers <= N_LAYERS:
            raise ValueError("n_layers must be 0 to %d, got %r" % (N_LAYERS, n_layers))
        L = feature_lengths(wav.shape[1], pad)
        if L[-1] < 1:
            raise ValueError("the audio is too short for one frame: %d samples (+ %d padding on each side); at least "
                             "400 are needed" % (wav.shape[1], pad))
        x = wav.detach().float().contiguous()
        dev = x.device
        P = self._pack(dev, n_layers, proj)
        B, T = x.shape[0], L[-1]
        La = 64 * -(-L[0] // 64)                                    # even at every one of the six halvings
        with torch.no_grad(), _Gemm("3xtf32") as G:
            y, part, L0 = ops.hubert_conv0(x, P["conv0"], pad, La)
            scale, shift = ops.hubert_gn_finalize(part, L0, *P["gn"])
            a = ops.hubert_act(y, scale, shift)
            for i, (w01, w2) in enumerate(P["convs"]):
                pairs = tuple(t.view(-1, 2 * C_FEAT) for t in a)    # row pairs [B La / 2, 1024]: a view, no copy
                out = G.mm(pairs, w01)
                if w2 is not None:                                  # + x[2t + 2] w2^T: the next pair's first half
                    nxt = tuple(t[1:, :C_FEAT] for t in pairs)
                    _mm_acc(out[:-1], nxt, w2)
                La //= 2
                y = out.view(B, La, C_FEAT)
                if i < 5:
                    a = ops.hubert_act(y)
                else:
                    _, a = ops.hubert_ln(y, *P["fp_norm"], T, gelu=True, h=False)
            h = G.mm(a, *P["fp"])
            pos = ops.hubert_posconv(h, *P["pos"], T)
            h, op = ops.hubert_ln(h, *P["norm"], T, y=pos, h=h)
            for j, lp in enumerate(P["layers"]):
                qkv = G.mm(op, *lp["qkv"])
                att = G.mm(ops.hubert_attention(qkv, T), *lp["out"])
                h, op = ops.hubert_ln(h, lp["n1"][0], lp["n1"][1], T, y=att, eps=lp["n1"][2], h=h)
                f = ops.hubert_act(G.mm(op, *lp["fc1"]))
                last = j == len(P["layers"]) - 1
                h, op = ops.hubert_ln(h, lp["n2"][0], lp["n2"][1], T, y=G.mm(f, *lp["fc2"]), eps=lp["n2"][2], h=h,
                                      operand=not last or proj)
            if proj:
                if op is None:                                      # no transformer layer ran
                    op = _split(h)
                h = G.mm(op, *P["proj"])
        return h.view(B, T, -1)

    def encode(self, x, layer=None):
        self._check(x)
        return self._run(x.reshape(x.shape[0], -1), 0, N_LAYERS if layer is None else layer), None

    def units(self, wav):
        self._check(wav)
        return self._run(wav.reshape(wav.shape[0], -1), UNITS_PAD, N_LAYERS, proj=True)


def _mm_acc(out, xs, w):
    """out += xs w^T in 3xTF32 (xs and w as TF32 halves)"""
    (xh, xl), (wh, wl) = xs, w
    out.addmm_(xh, wh.t()).addmm_(xl, wh.t()).addmm_(xh, wl.t())


# ---- fairseq checkpoints without fairseq -------------------------------------------------------------------------------
class _Inert:
    """stand-in for any fairseq.* / omegaconf.* global in a checkpoint: accepts whatever the pickle hands it"""

    def __init__(self, *args, **kwargs):
        self.__dict__["_args"] = args

    def __setstate__(self, state):
        self.__dict__["_state"] = state


_SAFE_BUILTINS = {"object", "dict", "list", "tuple", "set", "frozenset", "int", "float", "complex", "str", "bytes",
                  "bytearray", "bool", "slice"}
_SAFE_GLOBALS = {("collections", "OrderedDict"), ("collections", "defaultdict"), ("argparse", "Namespace"),
                 ("copyreg", "_reconstructor"), ("_codecs", "encode"), ("typing", "Any"), ("torch", "Size"),
                 ("torch._tensor", "_rebuild_from_type_v2"), ("torch.nn.parameter", "Parameter"),
                 ("numpy", "dtype"), ("numpy", "ndarray"), ("numpy.core.multiarray", "scalar"),
                 ("numpy.core.multiarray", "_reconstruct"), ("numpy._core.multiarray", "scalar"),
                 ("numpy._core.multiarray", "_reconstruct")}


class _RestrictedUnpickler(pickle.Unpickler):
    """fairseq.* / omegaconf.* globals become inert placeholders; besides them only the builtins, containers, numpy and
    torch tensor / storage / dtype rebuilders a checkpoint holds resolve.  Any other global (a callable such as
    os.system) raises UnpicklingError naming it."""

    def find_class(self, module, name):
        if module.split(".")[0] in ("fairseq", "omegaconf"):
            return type(name, (_Inert,), {"__module__": "ddsp_svc_b200.hubert._inert." + module})
        module = _compat_pickle.IMPORT_MAPPING.get(module, module)          # protocol 0-2 names (copy_reg, __builtin__)
        ok = ((module, name) in _SAFE_GLOBALS or (module == "builtins" and name in _SAFE_BUILTINS)
              or (module == "torch._utils" and name.startswith("_rebuild_"))
              or (module == "torch" and (name.endswith("Storage") or isinstance(getattr(torch, name, None), torch.dtype))))
        if not ok:
            raise pickle.UnpicklingError("the checkpoint refers to the global %s.%s, which a fairseq HuBERT checkpoint "
                                         "does not need; refusing to load it" % (module, name))
        return super().find_class(module, name)


_pickle_module = types.ModuleType("ddsp_svc_b200.hubert._pickle")
_pickle_module.Unpickler = _RestrictedUnpickler
_pickle_module.load = lambda f, **kw: _RestrictedUnpickler(f, **kw).load()
_pickle_module.__dict__.update({k: getattr(pickle, k) for k in ("HIGHEST_PROTOCOL", "dumps", "dump", "loads")})

_IGNORED_KEYS = ("mask_emb", "label_embs_concat")
_LAYER = r"encoder\.layers\.(\d+)\."
_RENAMES = [(r"feature_extractor\.conv_layers\.(\d)\.0\.weight", r"feature_extractor.conv\1.weight"),
            (r"feature_extractor\.conv_layers\.0\.2\.(weight|bias)", r"feature_extractor.norm0.\1"),
            (r"layer_norm\.(weight|bias)", r"feature_projection.norm.\1"),
            (r"post_extract_proj\.(weight|bias)", r"feature_projection.projection.\1"),
            (r"encoder\.pos_conv\.0\.(weight_g|weight_v|bias)", r"positional_embedding.conv.\1"),
            (r"encoder\.pos_conv\.0\.parametrizations\.weight\.original0", r"positional_embedding.conv.weight_g"),
            (r"encoder\.pos_conv\.0\.parametrizations\.weight\.original1", r"positional_embedding.conv.weight_v"),
            (r"encoder\.layer_norm\.(weight|bias)", r"norm.\1"),
            (_LAYER + r"self_attn\.out_proj\.(weight|bias)", r"encoder.layers.\1.self_attn.out_proj.\2"),
            (_LAYER + r"self_attn_layer_norm\.(weight|bias)", r"encoder.layers.\1.norm1.\2"),
            (_LAYER + r"final_layer_norm\.(weight|bias)", r"encoder.layers.\1.norm2.\2"),
            (_LAYER + r"fc1\.(weight|bias)", r"encoder.layers.\1.linear1.\2"),
            (_LAYER + r"fc2\.(weight|bias)", r"encoder.layers.\1.linear2.\2"),
            (r"final_proj\.(weight|bias)", r"proj.\1")]
_QKV = re.compile(_LAYER + r"self_attn\.([qkv])_proj\.(weight|bias)")


def _arch_fields(state):
    """the model's architecture fields from cfg['model'] or args, when readable -> dict (empty otherwise)"""
    cfg = state.get("cfg")
    src = cfg.get("model") if isinstance(cfg, collections.abc.Mapping) else None
    if src is None and isinstance(state.get("args"), argparse.Namespace):
        src = state["args"]
    if isinstance(src, argparse.Namespace):
        return vars(src)
    return dict(src) if isinstance(src, collections.abc.Mapping) else {}


def check_fairseq_arch(fields):
    """raise ValueError naming the field of a fairseq configuration the kernels do not implement"""
    def bad(name, want, got):
        raise ValueError("%s: only %r (HuBERT-base) is implemented, got %r" % (name, want, got))

    if fields.get("layer_norm_first", False):
        bad("layer_norm_first", False, fields["layer_norm_first"])
    if fields.get("extractor_mode", "default") != "default":
        bad("extractor_mode", "default", fields["extractor_mode"])
    cfl = fields.get("conv_feature_layers")
    if cfl is not None and re.sub(r"\s", "", str(cfl)) != CONV_FEATURE_LAYERS:
        bad("conv_feature_layers", CONV_FEATURE_LAYERS, cfl)
    for name, want in (("encoder_embed_dim", D_MODEL), ("encoder_attention_heads", N_HEADS), ("conv_pos", POS_TAPS),
                       ("conv_pos_groups", POS_GROUPS), ("encoder_layers", N_LAYERS), ("encoder_ffn_embed_dim", D_FFN)):
        if name in fields and fields[name] is not None and int(fields[name]) != want:
            bad(name, want, fields[name])


def _check_shapes(sd):
    """the architecture facts against the weight shapes (the mapped dict)"""
    want = {"feature_extractor.conv0.weight": ((C_FEAT, 1, 10), "conv_feature_layers"),
            "feature_projection.projection.weight": ((D_MODEL, C_FEAT), "encoder_embed_dim"),
            "positional_embedding.conv.weight_v": ((D_MODEL, D_MODEL // POS_GROUPS, POS_TAPS),
                                                   "conv_pos / conv_pos_groups"),
            "positional_embedding.conv.weight_g": ((1, 1, POS_TAPS), "conv_pos")}
    for i in range(1, 7):
        want["feature_extractor.conv%d.weight" % i] = ((C_FEAT, C_FEAT, 3 if i <= 4 else 2), "conv_feature_layers")
    for i in range(N_LAYERS):
        want["encoder.layers.%d.self_attn.in_proj_weight" % i] = ((3 * D_MODEL, D_MODEL), "encoder_embed_dim")
        want["encoder.layers.%d.linear1.weight" % i] = ((D_FFN, D_MODEL), "encoder_ffn_embed_dim")
    for k, (shape, field) in want.items():
        if k in sd and tuple(sd[k].shape) != shape:
            raise ValueError("%s: the weight %s has shape %s, the kernels implement %s"
                             % (field, k, tuple(sd[k].shape), shape))


def fairseq_to_hubert_state_dict(model_sd):
    """a fairseq HubertModel state dict -> HubertSoft's keys (q, k, v concatenated into in_proj_*), fp32.  Raises
    ValueError listing any key it does not know."""
    out, qkv, unknown = {}, {}, []
    for k, v in model_sd.items():
        if k in _IGNORED_KEYS:
            continue
        if torch.is_tensor(v) and v.is_floating_point():
            v = v.float()
        m = _QKV.fullmatch(k)
        if m:
            qkv.setdefault((int(m.group(1)), m.group(3)), {})[m.group(2)] = v
            continue
        for pat, rep in _RENAMES:
            if re.fullmatch(pat, k):
                out[re.sub(pat, rep, k)] = v
                break
        else:
            unknown.append(k)
    for (i, kind), parts in sorted(qkv.items()):
        if set(parts) != {"q", "k", "v"}:
            unknown.extend("encoder.layers.%d.self_attn.%s_proj.%s (q, k and v must all be present)" % (i, p, kind)
                           for p in parts)
            continue
        out["encoder.layers.%d.self_attn.in_proj_%s" % (i, kind)] = torch.cat([parts["q"], parts["k"], parts["v"]])
    if unknown:
        raise ValueError("unexpected keys in the fairseq checkpoint: %s" % ", ".join(sorted(unknown)))
    return out


def load_fairseq_hubert(path):
    """a fairseq HuBERT-base / ContentVec checkpoint -> HubertSoft in eval mode (CPU), without fairseq"""
    state = torch.load(path, map_location="cpu", pickle_module=_pickle_module, weights_only=False)
    if not isinstance(state, collections.abc.Mapping) or not isinstance(state.get("model"), collections.abc.Mapping):
        raise ValueError("%s is not a fairseq checkpoint (no 'model' state dict)" % (path,))
    check_fairseq_arch(_arch_fields(state))
    sd = fairseq_to_hubert_state_dict(state["model"])
    _check_shapes(sd)
    model = HubertSoft()
    if "proj.weight" in sd and sd["proj.weight"].shape != model.proj.weight.shape:
        model.proj = nn.Linear(*reversed(sd["proj.weight"].shape))
    unused = {"masked_spec_embed", "label_embedding.weight"}     # bshall's training-only parameters
    missing = sorted(set(model.state_dict()) - set(sd) - unused)
    if missing:
        raise ValueError("keys missing from the fairseq checkpoint (as HubertSoft names them): %s" % ", ".join(missing))
    unexpected = sorted(set(sd) - set(model.state_dict()))
    if unexpected:                              # e.g. the layers of a deeper checkpoint whose config was not readable
        raise ValueError("keys of the fairseq checkpoint that HubertSoft does not have: %s" % ", ".join(unexpected))
    model.load_state_dict(sd, strict=False)
    return model.eval()


# ---- Units_Encoder -----------------------------------------------------------------------------------------------------
class Units_Encoder:
    """The reference's Units_Encoder (ddsp/vocoder.py): Units_Encoder(encoder, encoder_ckpt, encoder_sample_rate=16000,
    encoder_hop_size=320, device=None).  encode(audio [B, N] CUDA, sample_rate, hop_size) -> units [1, n_frames, C]
    (frame f at row round(ratio f), as the reference gathers batch row 0).  encode_batch(audio [B, N], sample_rate,
    hop_size) -> [B, n_frames, C] on the device without syncs, every row encoded on its own."""

    def __init__(self, encoder, encoder_ckpt, encoder_sample_rate=16000, encoder_hop_size=320, device=None,
                 cnhubertsoft_gate=10):
        if encoder in ("hubertlarge1024l24", "cnhubertsoftfish"):
            raise ValueError("units encoder %r is not implemented on the kernels (%s)" % (
                encoder, "HuBERT-large: 1024 channels, 24 layers, pre-LN" if encoder == "hubertlarge1024l24" else
                "the transformers chinese-hubert-base with top-k gating"))
        if encoder not in KINDS:
            raise ValueError(f" [x] Unknown units encoder: {encoder}")
        device = torch.device("cuda" if device is None else device)
        if device.type != "cuda":
            raise ValueError("the units encoder runs on the CUDA kernels: device must be a CUDA device, got %s" % device)
        self.device = device
        self.encoder = encoder
        self.n_layers, self.proj, self.flatten = KINDS[encoder]
        if encoder == "hubertsoft":
            print(' [Encoder Model] HuBERT Soft')
            print(' [Loading] ' + encoder_ckpt)
            model = HubertSoft()
            ckpt = torch.load(encoder_ckpt, map_location="cpu")
            consume_prefix_in_state_dict_if_present(ckpt, "module.")
            model.load_state_dict(ckpt)
            self.pad = UNITS_PAD
        else:
            print(' [Encoder Model] %s' % ("Content Vec" if encoder.startswith("contentvec") else "HuBERT Base"))
            print(' [Loading] ' + encoder_ckpt)
            model = load_fairseq_hubert(encoder_ckpt)
            self.pad = 0
        self.model = model.eval().to(device)
        self._resampler = Resampler(encoder_sample_rate)
        self.resample_kernel = self._resampler.tables
        self.encoder_sample_rate = encoder_sample_rate
        self.encoder_hop_size = encoder_hop_size

    def _resample(self, audio, sample_rate):
        return self._resampler(audio, sample_rate)

    def _units(self, audio, sample_rate, flatten):
        if not (isinstance(audio, torch.Tensor) and audio.is_cuda):
            raise ValueError("the units encoder runs on the CUDA kernels: audio must be a CUDA tensor")
        if audio.dim() != 2:
            raise ValueError("audio must be [B, N], got %s" % (tuple(audio.shape),))
        audio = audio.detach().float().contiguous()
        audio_res = self._resample(audio, int(sample_rate))
        if audio_res.size(-1) < 400:                           # the reference pads the audio before resampling
            audio_res = F.pad(audio, (0, 400 - audio_res.size(-1)))
        if flatten:
            audio_res = audio_res.reshape(1, -1)
        with torch.no_grad():
            return self.model._run(audio_res, self.pad, self.n_layers, self.proj)

    def _ratio(self, sample_rate, hop_size):
        return (hop_size / sample_rate) / (self.encoder_hop_size / self.encoder_sample_rate)

    def encode(self, audio, sample_rate, hop_size):
        units = self._units(audio, sample_rate, self.flatten)
        n_frames = audio.size(-1) // hop_size + 1
        return ops.hubert_align(units[:1], self._ratio(sample_rate, hop_size), n_frames)

    def encode_batch(self, audio, sample_rate, hop_size):
        units = self._units(audio, sample_rate, False)
        n_frames = audio.size(-1) // hop_size + 1
        return ops.hubert_align(units, self._ratio(sample_rate, hop_size), n_frames)
