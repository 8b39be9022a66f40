"""Plain-torch restatement of the units-encoder path (reference ddsp/vocoder.py Units_Encoder.encode; HubertSoft in
encoder/hubert/model.py; fairseq's HubertModel.extract_features) over a ``ddsp_svc_b200.HubertSoft``'s state dict, in
any dtype and on any device: float64 is the comparator of the GPU tests, fp32 on CUDA under torch's defaults (cuDNN
TF32 convolutions, fp32 Linear) is what the reference runs and the eager arm of bench_units.py.

Resampling goes through tests/rmvpe_oracle.resample (the same torchaudio table, pinned there against torchaudio)."""
import argparse
import math
import sys
import types

import torch
import torch.nn.functional as F

from tests import rmvpe_oracle

KINDS = {"hubertsoft": (12, True, False),
         "hubertbase": (9, True, False), "hubertbase768": (9, False, False), "hubertbase768l12": (12, False, False),
         "contentvec": (9, True, True), "contentvec768": (9, False, True), "contentvec768l12": (12, False, True)}


def _layer(sd, i, x, dtype):
    g = lambda k: sd["encoder.layers.%d.%s" % (i, k)].to(x.device, dtype)
    B, T, D = x.shape
    qkv = F.linear(x, g("self_attn.in_proj_weight"), g("self_attn.in_proj_bias"))
    q, k, v = (t.reshape(B, T, 12, 64).transpose(1, 2) for t in qkv.split(D, -1))
    p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(64), -1)
    a = (p @ v).transpose(1, 2).reshape(B, T, D)
    x = F.layer_norm(x + F.linear(a, g("self_attn.out_proj.weight"), g("self_attn.out_proj.bias")), (D,),
                     g("norm1.weight"), g("norm1.bias"), 1e-5)
    f = F.linear(F.gelu(F.linear(x, g("linear1.weight"), g("linear1.bias"))), g("linear2.weight"), g("linear2.bias"))
    return F.layer_norm(x + f, (D,), g("norm2.weight"), g("norm2.bias"), 1e-5)


def features(sd, wav, dtype=torch.float64):
    """feature extractor + feature projection of wav [B, N] -> [B, T, 768]"""
    g = lambda k: sd[k].to(wav.device, dtype)
    x = F.conv1d(wav.to(dtype)[:, None], g("feature_extractor.conv0.weight"), stride=5)
    x = F.gelu(F.group_norm(x, 512, g("feature_extractor.norm0.weight"), g("feature_extractor.norm0.bias"), 1e-5))
    for i in range(1, 7):
        x = F.gelu(F.conv1d(x, g("feature_extractor.conv%d.weight" % i), stride=2))
    x = F.layer_norm(x.transpose(1, 2), (512,), g("feature_projection.norm.weight"), g("feature_projection.norm.bias"),
                     1e-5)
    return F.linear(x, g("feature_projection.projection.weight"), g("feature_projection.projection.bias"))


def positional(sd, x, dtype=torch.float64):
    """GELU(weight-normed grouped Conv1d(768, 768, 128, padding 64, groups 16)(x)[..., :-1]) of x [B, T, 768]"""
    g = lambda k: sd[k].to(x.device, dtype)
    w = torch._weight_norm(g("positional_embedding.conv.weight_v"), g("positional_embedding.conv.weight_g"), 2)
    y = F.conv1d(x.transpose(1, 2), w, g("positional_embedding.conv.bias"), padding=64, groups=16)
    return F.gelu(y[:, :, :-1]).transpose(1, 2)


def encode(sd, wav, n_layers=12, proj=False, pad=0, dtype=torch.float64):
    """wav [B, N] zero-padded by `pad` on each side -> [B, T, 768] after n_layers post-LN layers (proj: [B, T, 256])"""
    wav = F.pad(wav.to(dtype), (pad, pad))
    x = features(sd, wav, dtype)
    g = lambda k: sd[k].to(x.device, dtype)
    x = F.layer_norm(x + positional(sd, x, dtype), (768,), g("norm.weight"), g("norm.bias"), 1e-5)
    for i in range(n_layers):
        x = _layer(sd, i, x, dtype)
    return F.linear(x, g("proj.weight"), g("proj.bias")) if proj else x


def units(sd, wav, dtype=torch.float64):
    """HubertSoft.units of wav [B, N]: the 40-sample pad on each side, 12 layers, proj"""
    return encode(sd, wav, 12, True, 40, dtype)


def align_index(n_frames, ratio, T, device="cpu"):
    """the reference's index: clamp(round(ratio * arange(n_frames)).long(), max=T - 1), in torch's float32"""
    return torch.clamp(torch.round(ratio * torch.arange(n_frames).to(device)).long(), max=T - 1)


def units_encode(kind, sd, audio, sample_rate, hop_size, dtype=torch.float64, encoder_hop_size=320, batch=False,
                 tabs=None):
    """Units_Encoder(kind).encode(audio [B, N], sample_rate, hop_size) -> [1, n_frames, C] (batch: every row on its
    own, [B, n_frames, C], as Units_Encoder.encode_batch).  tabs: rmvpe_oracle.tables(sample_rate, ...) built once, as
    the reference caches its Resample per rate (built on every call when None)"""
    n_layers, proj, flatten = KINDS[kind]
    audio_res = rmvpe_oracle.resample(audio, sample_rate, dtype, tabs)
    if audio_res.size(-1) < 400:
        audio_res = F.pad(audio.to(dtype), (0, 400 - audio_res.size(-1)))
    if flatten and not batch:
        audio_res = audio_res.reshape(1, -1)
    u = encode(sd, audio_res, n_layers, proj, 40 if kind == "hubertsoft" else 0, dtype)
    n_frames = audio.size(-1) // hop_size + 1
    ratio = (hop_size / sample_rate) / (encoder_hop_size / 16000)
    index = align_index(n_frames, ratio, u.size(1), u.device)
    if batch:
        return u[:, index]
    return torch.gather(u, 1, index.unsqueeze(0).unsqueeze(-1).repeat([1, 1, u.size(-1)]))


def seeded_state_dict(seed=0, peaked=False):
    """a HubertSoft state dict drawn from a seed (float32 CPU): weights scaled so every layer's output stays O(1), the
    GroupNorm and LayerNorm affines near identity.  peaked: q and k projections scaled 2x so attention rows are
    dominated by a few keys (max probability > 0.5)"""
    from ddsp_svc_b200.hubert import HubertSoft
    g = torch.Generator().manual_seed(seed)
    shapes = {k: v.shape for k, v in HubertSoft().state_dict().items()}
    sd = {}
    for k, shape in shapes.items():
        parts = k.split(".")
        if len(parts) > 1 and "norm" in parts[-2] and parts[-1] == "weight":
            v = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif k.endswith("bias"):
            v = 0.1 * torch.randn(shape, generator=g)
        elif k.endswith("weight_g"):
            v = 1.0 + 0.1 * torch.rand(shape, generator=g)
        else:
            fan_in = shape[1] * (shape[2] if len(shape) > 2 else 1) if len(shape) > 1 else 1
            v = torch.randn(shape, generator=g) / math.sqrt(fan_in)
        sd[k] = v.float()
    if peaked:
        for i in range(12):
            sd["encoder.layers.%d.self_attn.in_proj_weight" % i][:1536] *= 2.0
    return sd


# ---- synthetic fairseq checkpoints ---------------------------------------------------------------------------------------
def fairseq_state_dict(seed=0, final_rows=256):
    """a synthetic fairseq HubertModel state dict (float16 where fairseq stores half, as some checkpoints do)"""
    sd = seeded_state_dict(seed)
    out = {"mask_emb": torch.zeros(768), "label_embs_concat": torch.zeros(504, 256)}
    for i in range(7):
        out["feature_extractor.conv_layers.%d.0.weight" % i] = sd["feature_extractor.conv%d.weight" % i].half()
    out["feature_extractor.conv_layers.0.2.weight"] = sd["feature_extractor.norm0.weight"]
    out["feature_extractor.conv_layers.0.2.bias"] = sd["feature_extractor.norm0.bias"]
    for a, b in (("layer_norm", "feature_projection.norm"), ("post_extract_proj", "feature_projection.projection"),
                 ("encoder.layer_norm", "norm")):
        out[a + ".weight"], out[a + ".bias"] = sd[b + ".weight"], sd[b + ".bias"]
    for p in ("weight_g", "weight_v", "bias"):
        out["encoder.pos_conv.0." + p] = sd["positional_embedding.conv." + p]
    for i in range(12):
        f, t = "encoder.layers.%d." % i, "encoder.layers.%d." % i
        for kind in ("weight", "bias"):
            q, k, v = sd[t + "self_attn.in_proj_" + kind].chunk(3)
            out[f + "self_attn.q_proj." + kind], out[f + "self_attn.k_proj." + kind] = q, k
            out[f + "self_attn.v_proj." + kind] = v
            out[f + "self_attn.out_proj." + kind] = sd[t + "self_attn.out_proj." + kind]
            out[f + "self_attn_layer_norm." + kind] = sd[t + "norm1." + kind]
            out[f + "final_layer_norm." + kind] = sd[t + "norm2." + kind]
            out[f + "fc1." + kind] = sd[t + "linear1." + kind]
            out[f + "fc2." + kind] = sd[t + "linear2." + kind]
    out["final_proj.weight"] = torch.randn(final_rows, 768) / 28.0
    out["final_proj.bias"] = torch.zeros(final_rows)
    return sd, out


class _FakeFairseqTask:                                          # pickled under a fairseq.* module name below
    def __init__(self):
        self.name = "hubert_pretraining"


def save_fairseq(path, model_sd, args=None, cfg=None):
    """torch.save a fairseq-style checkpoint whose task_state is an instance of a class pickled as a fairseq.* global"""
    names = ("fairseq", "fairseq.tasks", "fairseq.tasks.hubert_pretraining")
    added = [n for n in names if n not in sys.modules]
    for n in added:
        sys.modules[n] = types.ModuleType(n)
    leaf = sys.modules[names[-1]]
    _FakeFairseqTask.__module__ = leaf.__name__
    _FakeFairseqTask.__qualname__ = "HubertPretrainingTask"
    leaf.HubertPretrainingTask = _FakeFairseqTask
    try:
        state = {"model": model_sd, "args": args, "cfg": cfg, "task_state": _FakeFairseqTask()}
        torch.save(state, path)
    finally:
        del leaf.HubertPretrainingTask
        for n in added:
            del sys.modules[n]
        _FakeFairseqTask.__module__ = __name__
        _FakeFairseqTask.__qualname__ = "_FakeFairseqTask"


def fairseq_args(**kw):
    a = dict(layer_norm_first=False, extractor_mode="default", encoder_embed_dim=768, encoder_attention_heads=12,
             conv_pos=128, conv_pos_groups=16, encoder_layers=12, encoder_ffn_embed_dim=3072,
             conv_feature_layers="[(512,10,5)] + [(512,3,2)] * 4 + [(512,2,2)] * 2")
    a.update(kw)
    return argparse.Namespace(**a)
