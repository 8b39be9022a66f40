"""The units encoder on the GPU against the float64 oracle (tests/units_oracle.py): every launch kind of csrc/hubert.cu,
the whole encoder for HubertSoft and the fairseq layer-9 / layer-12 configurations, Units_Encoder.encode at 16 and
44.1 kHz, determinism, and a sync-free warm encode_batch."""

import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import hubert as H
from ddsp_svc_b200 import ops
from tests import units_oracle as U

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(got, want):
    want = want.double().cpu()
    return ((got.double().cpu() - want).norm() / want.norm()).item()


def _gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.fixture(scope="module")
def soft():
    sd = U.seeded_state_dict(11)
    m = H.HubertSoft()
    m.load_state_dict(sd)
    return sd, m.eval().to(DEV)


@pytest.mark.parametrize("N,pad", [(400, 40), (16000, 40), (8000, 0)])
def test_conv0_groupnorm(soft, N, pad):
    sd, m = soft
    x = torch.randn(2, N, generator=_gen(N))
    P = m._pack(torch.device(DEV), 12, True)
    L0 = (N + 2 * pad - 10) // 5 + 1
    La = 64 * -(-L0 // 64)
    y, part, l0 = ops.hubert_conv0(x.to(DEV), P["conv0"], pad, La)
    assert l0 == L0 and torch.all(y[:, L0:] == 0)
    scale, shift = ops.hubert_gn_finalize(part, L0, *P["gn"])
    got = ops.hubert_act(y, scale, shift, split=False)[:, :L0]
    c = F.conv1d(F.pad(x.double(), (pad, pad))[:, None], sd["feature_extractor.conv0.weight"].double(), stride=5)
    want = F.gelu(F.group_norm(c, 512, sd["feature_extractor.norm0.weight"].double(),
                               sd["feature_extractor.norm0.bias"].double(), 1e-5)).transpose(1, 2)
    assert rel(got, want) < 2e-6


def test_conv0_silent_clip(soft):
    sd, m = soft
    P = m._pack(torch.device(DEV), 12, True)
    y, part, L0 = ops.hubert_conv0(torch.zeros(1, 1600, device=DEV), P["conv0"], 40, 384)
    scale, shift = ops.hubert_gn_finalize(part, L0, *P["gn"])
    got = ops.hubert_act(y, scale, shift, split=False)[:, :L0]
    want = F.gelu(sd["feature_extractor.norm0.bias"].double())
    assert torch.allclose(got.double().cpu(), want.expand_as(got.cpu()), rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 500, 2999])
def test_attention(T):
    B = 2 if T < 1000 else 1
    qkv = torch.randn(B * T, 2304, generator=_gen(T)) * 1.5
    o = ops.hubert_attention(qkv.to(DEV), T, split=False)
    q, k, v = (t.double().view(B, T, 12, 64).transpose(1, 2) for t in qkv.split(768, -1))
    p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1)
    want = (p @ v).transpose(1, 2).reshape(B * T, 768)
    assert rel(o, want) < 3e-6
    hi, lo = ops.hubert_attention(qkv.to(DEV), T)
    assert rel(hi + lo, want) < 3e-6


def test_attention_peaked():
    T = 300
    qkv = torch.randn(T, 2304, generator=_gen(5))
    qkv[:, :768] *= 8.0
    q, k, v = (t.double().view(1, T, 12, 64).transpose(1, 2) for t in qkv.split(768, -1))
    p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1)
    assert p.max(-1).values.median() > 0.5
    want = (p @ v).transpose(1, 2).reshape(T, 768)
    assert rel(ops.hubert_attention(qkv.to(DEV), T, split=False), want) < 3e-6


@pytest.mark.parametrize("T", [1, 37, 499])
def test_posconv(soft, T):
    sd, m = soft
    P = m._pack(torch.device(DEV), 12, True)
    x = torch.randn(2, T, 768, generator=_gen(T))
    got = ops.hubert_posconv(x.view(-1, 768).to(DEV), *P["pos"], T)
    want = U.positional(sd, x.double()).reshape(-1, 768)
    assert rel(got, want) < 2e-6


@pytest.mark.parametrize("C,gelu", [(768, False), (512, True)])
def test_add_layernorm(C, gelu):
    B, T, rows_per_b = 2, 50, (50 if C == 768 else 64)
    x = torch.randn(B, rows_per_b, C, generator=_gen(C)) * 3 + 1
    y = torch.randn(B * T, C, generator=_gen(C + 1)) if not gelu else None
    g, b = torch.rand(C, generator=_gen(1)) + 0.5, torch.randn(C, generator=_gen(2))
    h, (hi, lo) = ops.hubert_ln(x.to(DEV), g.to(DEV), b.to(DEV), T, y=None if y is None else y.to(DEV), gelu=gelu)
    v = x[:, :T].double().reshape(B * T, C)
    if y is not None:
        v = v + y.double()
    if gelu:
        v = F.gelu(v)
    want = F.layer_norm(v, (C,), g.double(), b.double(), 1e-5)
    assert rel(h, want) < 1e-6
    assert torch.equal(hi + lo, h) or rel(hi + lo, want) < 1e-6


@pytest.mark.parametrize("sr,hop", [(44100, 512), (16000, 320)])
def test_align(sr, hop):
    n_frames, T = 200000, 200000               # no clamping: the 197 frames where a float64 index differs are compared
    ratio = (hop / sr) / (320 / 16000)
    units = torch.arange(T, dtype=torch.float32, device=DEV).view(1, T, 1)
    got = ops.hubert_align(units, ratio, n_frames).view(-1).long().cpu()
    assert torch.equal(got, U.align_index(n_frames, ratio, T))


def _encoder_bounds(got, want):
    e = rel(got, want)
    print("rel rms %.3e" % e)
    assert e < 4e-5                                             # measured up to 1.6e-5 (H100 80GB HBM3, 700 W)
    return e


@pytest.mark.parametrize("N,B", [(400, 1), (8000, 3), (32000, 1), (160000, 1)])
def test_hubertsoft_units(soft, N, B):
    sd, m = soft
    wav = torch.randn(B, N, generator=_gen(N + B)) * 0.3
    with torch.no_grad():
        got = m.units(wav[:, None].to(DEV))
    want = U.units(sd, wav)
    _encoder_bounds(got, want)


@pytest.mark.parametrize("layer,proj", [(9, False), (12, False), (9, True)])
@pytest.mark.parametrize("N,B", [(8000, 1), (24000, 3)])
def test_fairseq_layers(layer, proj, N, B):
    sd = U.seeded_state_dict(12 + layer, peaked=layer == 12)
    m = H.HubertSoft()
    m.load_state_dict(sd)
    m = m.eval().to(DEV)
    wav = torch.randn(B, N, generator=_gen(N)) * 0.3
    got = m._run(wav.to(DEV), 0, layer, proj)
    want = U.encode(sd, wav, layer, proj)
    _encoder_bounds(got, want)


@pytest.fixture(scope="module")
def encoders(tmp_path_factory):
    d = tmp_path_factory.mktemp("ckpt")
    sd = U.seeded_state_dict(21)
    torch.save({"module." + k: v for k, v in sd.items()}, d / "soft.pt")
    fsd_sd, fsd = U.fairseq_state_dict(22)
    U.save_fairseq(d / "cv.pt", fsd, args=U.fairseq_args())
    ref_sd = H.load_fairseq_hubert(str(d / "cv.pt")).state_dict()
    return dict(soft=(str(d / "soft.pt"), sd), cv=(str(d / "cv.pt"), ref_sd))


@pytest.mark.parametrize("kind", ["hubertsoft", "contentvec768l12", "contentvec", "hubertbase768"])
@pytest.mark.parametrize("sr,hop,N,B", [(16000, 320, 16000, 1), (44100, 512, 44100, 1), (44100, 512, 1000, 1),
                                        (44100, 512, 22050, 2)])
def test_units_encoder_encode(encoders, kind, sr, hop, N, B):
    path, sd = encoders["soft" if kind == "hubertsoft" else "cv"]
    enc = H.Units_Encoder(kind, path, device=DEV)
    audio = torch.randn(B, N, generator=_gen(sr + N)) * 0.3
    got = enc.encode(audio.to(DEV), sr, hop)
    want = U.units_encode(kind, sd, audio, sr, hop)
    assert got.shape == want.shape
    _encoder_bounds(got, want)


def test_determinism_and_sync_free_encode_batch(encoders):
    path, sd = encoders["cv"]
    enc = H.Units_Encoder("contentvec768l12", path, device=DEV)
    audio = (torch.randn(3, 44100, generator=_gen(7)) * 0.3).to(DEV)
    a = enc.encode_batch(audio, 44100, 512)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = enc.encode_batch(audio, 44100, 512)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(a, b)
    want = U.units_encode("contentvec768l12", sd, audio.cpu(), 44100, 512, batch=True)
    _encoder_bounds(a, want)


def test_training_mode_under_grad_raises(soft):
    m = H.HubertSoft().to(DEV).train()
    with pytest.raises(NotImplementedError):
        m.units(torch.zeros(1, 1, 400, device=DEV))


@pytest.mark.parametrize("name", list(__import__("tests.golden.make_golden_units", fromlist=["CASES"]).CASES))
def test_golden_replay(name, tmp_path):
    from tests.golden import make_golden_units as mk
    d, sd = mk.load(name)
    x = torch.from_numpy(d["audio"]).to(DEV)
    if "sr" in d:
        path = tmp_path / "soft.pt"
        torch.save({"module." + k: v for k, v in sd.items()}, path)
        got = H.Units_Encoder("hubertsoft", str(path), device=DEV).encode(x, int(d["sr"]), int(d["hop"]))
    else:
        m = H.HubertSoft()
        m.load_state_dict(sd)
        got = m.eval().to(DEV).units(x[:, None])
    want = torch.from_numpy(d["units"]).double()
    assert got.shape == want.shape
    _encoder_bounds(got, want)
