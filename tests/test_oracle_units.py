"""CPU checks of the units-encoder oracle and of ddsp_svc_b200.hubert's host logic: the oracle against the reference's
HubertSoft and against transformers' HubertModel (fairseq semantics), the float32 alignment index, weight-norm
folding, the row-pair GEMM form of the strided convolutions, and the fairseq checkpoint loader."""
import argparse
import io
import pickle
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import hubert as H
from oracle import ref_loader
from tests import units_oracle as U


def _reference_hubert():
    ref_loader.load()
    if "sklearn.cluster" not in sys.modules:                   # encoder.hubert.model imports KMeans for HubertDiscrete
        try:
            import sklearn.cluster  # noqa: F401
        except ImportError:
            sys.modules.setdefault("sklearn", types.ModuleType("sklearn"))
            sys.modules["sklearn.cluster"] = types.SimpleNamespace(KMeans=object)
    from encoder.hubert import model
    return model


@pytest.mark.skipif(not ref_loader.available(), reason="needs the reference checkout (DDSP_REFERENCE_ROOT)")
@pytest.mark.parametrize("n,B", [(400, 1), (8000, 2)])
def test_oracle_matches_reference_hubertsoft(n, B):
    ref = _reference_hubert().HubertSoft()
    sd = U.seeded_state_dict(1)
    ref.load_state_dict(sd)
    ref = ref.double().eval()
    wav = torch.randn(B, n, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    with torch.inference_mode():
        want = ref.units(wav[:, None])
        got = U.units(sd, wav)
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("layer,proj", [(9, False), (12, False), (9, True)])
def test_oracle_matches_transformers_hubert_through_fairseq_mapping(layer, proj):
    transformers = pytest.importorskip("transformers")
    cfg = transformers.HubertConfig()                           # HuBERT-base, fairseq layout (post-LN, group norm)
    torch.manual_seed(3)
    hf = transformers.HubertModel(cfg).double().eval()
    fsd = _fairseq_from_transformers(hf.state_dict())
    final = torch.nn.Linear(768, 256).double()
    fsd["final_proj.weight"], fsd["final_proj.bias"] = final.weight.detach(), final.bias.detach()
    sd = H.fairseq_to_hubert_state_dict(fsd)
    wav = torch.randn(1, 6400, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    with torch.no_grad():
        want = hf(wav, output_hidden_states=True).hidden_states[layer]
        if proj:
            want = final(want)
        got = U.encode(sd, wav, layer, proj)
    assert torch.allclose(got, want, rtol=1e-7, atol=1e-7), (got - want).abs().max()


def _fairseq_from_transformers(hsd):
    """transformers' HubertModel keys -> fairseq's (the inverse of the mapping transformers' converter applies)"""
    out = {}
    for k, v in hsd.items():
        k2 = k
        for a, b in (("feature_extractor.conv_layers.0.layer_norm", "feature_extractor.conv_layers.0.2"),
                     ("feature_projection.layer_norm", "layer_norm"),
                     ("feature_projection.projection", "post_extract_proj"),
                     ("encoder.pos_conv_embed.conv", "encoder.pos_conv.0"),
                     ("attention.", "self_attn."), ("self_attn.out_proj", "self_attn.out_proj"),
                     ("layer_norm.", "self_attn_layer_norm.") if ".layers." in k and ".final_" not in k else ("", ""),
                     ("feed_forward.intermediate_dense", "fc1"), ("feed_forward.output_dense", "fc2"),
                     ("encoder.layer_norm", "encoder.layer_norm")):
            if a:
                k2 = k2.replace(a, b)
        import re
        k2 = re.sub(r"feature_extractor\.conv_layers\.(\d)\.conv\.weight", r"feature_extractor.conv_layers.\1.0.weight", k2)
        k2 = k2.replace("final_self_attn_layer_norm", "final_layer_norm")
        out[k2] = v
    pg = [k for k in out if "pos_conv.0.parametrizations" in k]
    for k in pg:
        out[k.replace("parametrizations.weight.original0", "weight_g").replace("parametrizations.weight.original1",
                                                                              "weight_v")] = out.pop(k)
    out.pop("masked_spec_embed", None)
    return out


@pytest.mark.parametrize("sr,hop", [(44100, 512), (16000, 320), (24000, 480), (32000, 320), (48000, 512),
                                    (44100, 441)])
def test_align_index_matches_torch_float32_formula(sr, hop):
    n = 200000
    ratio = (hop / sr) / (320 / 16000)
    want = U.align_index(n, ratio, 10 ** 9).numpy()
    got = H.align_index(n, ratio, 10 ** 9)
    assert np.array_equal(got, want)
    if (sr, hop) == (44100, 512):
        f64 = np.minimum(np.round(ratio * np.arange(n, dtype=np.float64)), 10 ** 9).astype(np.int64)
        assert got[113250] != f64[113250]                       # where a float64 index would differ


def test_fold_weight_norm_matches_torch():
    g = torch.rand(1, 1, 128, dtype=torch.float64) + 0.5
    v = torch.randn(768, 48, 128, dtype=torch.float64)
    assert torch.allclose(H.fold_weight_norm(g, v), torch._weight_norm(v, g, 2), rtol=1e-13, atol=0)


@pytest.mark.parametrize("k,L", [(3, 64), (3, 10), (2, 64), (2, 4)])
def test_row_pair_gemm_matches_conv1d(k, L):
    gen = torch.Generator().manual_seed(k * 100 + L)
    x = torch.randn(2, L, 512, generator=gen, dtype=torch.float64)       # channel-contiguous, L even
    w = torch.randn(512, 512, k, generator=gen, dtype=torch.float64)
    want = F.conv1d(x.transpose(1, 2), w, stride=2).transpose(1, 2)     # [2, (L - k) // 2 + 1, 512]
    w01, w2 = H.pack_strided_conv(w)
    P = x.reshape(-1, 1024)                                               # the row pairs of both utterances
    out = P @ w01.t()
    if w2 is not None:
        out[:-1] += P[1:, :512] @ w2.t()
    got = out.view(2, L // 2, 512)[:, :want.shape[1]]
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-10)


def test_posconv_packing_layout():
    w = torch.randn(768, 48, 128, dtype=torch.float64)
    p = H.pack_posconv(w)
    g, k, ci, co = 5, 17, 7, 40
    assert p[g, k, ci, co] == w[g * 48 + co, ci, k]


# ---- the fairseq loader ------------------------------------------------------------------------------------------------
def test_fairseq_checkpoint_loads_strict_without_fairseq(tmp_path):
    sd, fsd = U.fairseq_state_dict(5)
    path = tmp_path / "checkpoint_best_legacy_500.pt"
    U.save_fairseq(path, fsd, args=U.fairseq_args())
    assert "fairseq" not in sys.modules or not hasattr(sys.modules["fairseq"], "__file__")
    model = H.load_fairseq_hubert(str(path))
    got = model.state_dict()
    for k, v in sd.items():
        if k in ("masked_spec_embed", "label_embedding.weight", "proj.weight", "proj.bias"):
            continue
        want = v.half().float() if k.startswith("feature_extractor.conv") else v
        assert torch.equal(got[k], want), k
        assert got[k].dtype == torch.float32
    assert torch.equal(got["proj.weight"], fsd["final_proj.weight"])


def test_fairseq_cfg_dict_is_read(tmp_path):
    _, fsd = U.fairseq_state_dict(6)
    path = tmp_path / "c.pt"
    U.save_fairseq(path, fsd, cfg={"model": vars(U.fairseq_args(layer_norm_first=True))})
    with pytest.raises(ValueError, match="layer_norm_first"):
        H.load_fairseq_hubert(str(path))


@pytest.mark.parametrize("field,value", [("layer_norm_first", True), ("extractor_mode", "layer_norm"),
                                         ("conv_feature_layers", "[(512,10,5)] + [(512,3,2)] * 5"),
                                         ("encoder_embed_dim", 1024), ("encoder_attention_heads", 16),
                                         ("conv_pos", 64), ("conv_pos_groups", 8)])
def test_fairseq_configuration_errors_name_the_field(tmp_path, field, value):
    _, fsd = U.fairseq_state_dict(7)
    path = tmp_path / "c.pt"
    U.save_fairseq(path, fsd, args=U.fairseq_args(**{field: value}))
    with pytest.raises(ValueError, match=field):
        H.load_fairseq_hubert(str(path))


def test_fairseq_weight_shapes_are_checked():
    _, fsd = U.fairseq_state_dict(8)
    fsd["encoder.pos_conv.0.weight_v"] = torch.zeros(768, 96, 128)
    with pytest.raises(ValueError, match="conv_pos"):
        H._check_shapes(H.fairseq_to_hubert_state_dict(fsd))


def test_fairseq_unknown_and_missing_keys_raise(tmp_path):
    _, fsd = U.fairseq_state_dict(9)
    fsd["encoder.layers.0.extra.weight"] = torch.zeros(3)
    with pytest.raises(ValueError, match="encoder.layers.0.extra.weight"):
        H.fairseq_to_hubert_state_dict(fsd)
    _, fsd = U.fairseq_state_dict(9)
    del fsd["encoder.layers.11.fc2.bias"]
    path = tmp_path / "c.pt"
    U.save_fairseq(path, fsd, args=U.fairseq_args())
    with pytest.raises(ValueError, match="encoder.layers.11.linear2.bias"):
        H.load_fairseq_hubert(str(path))


def test_bshall_checkpoint_loads_strict():
    sd = U.seeded_state_dict(10)
    ckpt = {"module." + k: v for k, v in sd.items()}
    torch.nn.modules.utils.consume_prefix_in_state_dict_if_present(ckpt, "module.")
    model = H.HubertSoft()
    model.load_state_dict(ckpt, strict=True)


def test_restricted_unpickler_makes_fairseq_globals_inert():
    raw = pickle.dumps(argparse.Namespace(a=1), protocol=0).replace(b"argparse", b"fairseq.x")
    obj = H._RestrictedUnpickler(io.BytesIO(raw)).load()
    assert isinstance(obj, H._Inert)


def test_restricted_unpickler_refuses_other_callables():
    raw = pickle.dumps(argparse.Namespace(a=1), protocol=0).replace(b"argparse\nNamespace", b"os\nsystem")
    with pytest.raises(pickle.UnpicklingError, match="os.system"):
        H._RestrictedUnpickler(io.BytesIO(raw)).load()


def test_fairseq_deeper_checkpoint_raises_on_the_extra_layers(tmp_path):
    _, fsd = U.fairseq_state_dict(12)
    for k in [k for k in fsd if k.startswith("encoder.layers.11.")]:
        fsd[k.replace("layers.11.", "layers.12.")] = fsd[k].clone()
    path = tmp_path / "c.pt"
    U.save_fairseq(path, fsd)                                   # no readable config: only the keys can tell
    with pytest.raises(ValueError, match="encoder.layers.12.linear1.weight"):
        H.load_fairseq_hubert(str(path))


@pytest.mark.parametrize("encoder", ["hubertlarge1024l24", "cnhubertsoftfish"])
def test_unsupported_encoders_raise(encoder):
    with pytest.raises(ValueError, match="not implemented"):
        H.Units_Encoder(encoder, "unused.pt", device="cuda")


def test_cpu_device_raises(tmp_path):
    with pytest.raises(ValueError, match="CUDA"):
        H.Units_Encoder("hubertsoft", "unused.pt", device="cpu")


# ---- the oracle against the reference's goldens (tests/golden/make_golden_units.py) ------------------------------------
@pytest.mark.parametrize("name", list(__import__("tests.golden.make_golden_units", fromlist=["CASES"]).CASES))
def test_oracle_matches_golden(name):
    from tests.golden import make_golden_units as mk
    d, sd = mk.load(name)
    x = torch.from_numpy(d["audio"])
    if "sr" in d:
        got = U.units_encode("hubertsoft", sd, x, int(d["sr"]), int(d["hop"]))
    else:
        got = U.units(sd, x)
    want = torch.from_numpy(d["units"]).double()
    assert got.shape == want.shape
    assert ((got - want).norm() / want.norm()).item() < 1e-6        # the goldens are float64 results stored in fp32
