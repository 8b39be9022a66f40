"""The NSF-HiFiGAN oracle (tests/hifigan_oracle.py) against the reference's own outputs, and the host side of the
package's Generator: weight-norm folding, the kernel's weight packing, the polyphase transposed convolution, strict
state-dict loading and the configuration checks.  CPU only."""
import json
import os
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import hifigan
from tests import hifigan_oracle as ho
from tests.golden import make_golden_hifigan as mk

HERE = os.path.dirname(os.path.abspath(__file__))


def _generator(d):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")           # torch.nn.utils.weight_norm is deprecated; the reference uses it
        return hifigan.Generator(ho.config(d))


def _source64(sd, f0, rand_ini, noise, upp, sr=44100):
    """SourceModuleHnNSF in float64 with the given draws (sinegen.py's reference semantics)"""
    f0 = f0.double().unsqueeze(-1)
    rad = f0 / sr * torch.arange(1, upp + 1, dtype=torch.float64)
    rad2 = torch.fmod(rad[..., -1:].float() + 0.5, 1.0) - 0.5
    rad_acc = rad2.cumsum(dim=1).fmod(1.0).to(rad)
    rad += F.pad(rad_acc, (0, 0, 1, -1))
    rad = rad.reshape(f0.shape[0], -1, 1) * torch.arange(1, 10, dtype=torch.float64).reshape(1, 1, -1)
    sines = torch.sin(2 * np.pi * (rad + rand_ini.double())) * 0.1
    uv = (f0 > 0).double().repeat_interleave(upp, dim=1)
    amp = uv * 0.003 + (1 - uv) * 0.1 / 3
    s = sines * uv + amp * noise.double()
    return torch.tanh(s @ sd["m_source.l_linear.weight"].double().t() + sd["m_source.l_linear.bias"].double())


@pytest.mark.parametrize("name", list(mk.CASES))
def test_oracle_matches_the_reference_goldens(name):
    c = mk.CASES[name]
    d = np.load(mk.path(name))
    sd = mk.seeded_state_dict(c["model"])
    h = ho.config(mk.MODELS[c["model"]]["h"])
    # the reference removed weight norm in fp32 before .double(); with weight norm attached it folds in float64
    net = ho.build(h, sd, fold_dtype=torch.float64 if c.get("weight_norm") else torch.float32)
    x, f0 = torch.from_numpy(d["x"]), torch.from_numpy(d["f0"])
    rand_ini, noise = mk.draws(d)
    har = _source64(sd, f0, rand_ini, noise, net.upp)
    with torch.no_grad():
        out = net(x.double(), har)
    ref = torch.from_numpy(d["out64"])
    assert out.shape == ref.shape
    # 4e-8 at most here (the source restated above differs in the last bits), against 1e-6 to 3e-6 for the fp32 reference
    assert (out - ref).abs().max().item() < 1e-7
    assert (torch.from_numpy(d["out32"]).double() - ref).abs().max().item() < 1e-5


@pytest.mark.parametrize("u,c_in,c_out", [(8, 32, 16), (2, 16, 32), (4, 16, 16)])
def test_polyphase_packing_equals_conv_transpose(u, c_in, c_out):
    g = torch.Generator().manual_seed(u)
    w = torch.randn(c_in, c_out, 2 * u, generator=g).double()
    b = torch.randn(c_out, generator=g, dtype=torch.float64)
    for T in (1, 2, 9):
        x = torch.randn(2, c_in, T, generator=g, dtype=torch.float64)
        ref = F.conv_transpose1d(x, w, b, stride=u, padding=u // 2)
        wp = hifigan.pack_conv(hifigan.polyphase(w.float(), u))
        y = ho.packed_conv(x.transpose(1, 2), wp, torch.zeros(u * c_out), u * c_out, 3, 1)   # [B, T, u C_out]
        y = y.reshape(2, T * u, c_out).transpose(1, 2) + b[None, :, None]
        # hi + lo carries fp32 weights to 2^-22 relative (the TF32 split of the product is exact to that bound)
        assert y.shape == ref.shape and (y - ref).abs().max().item() < 1e-5


@pytest.mark.parametrize("k,d", [(3, 1), (7, 3), (11, 5), (7, 1)])
def test_packed_conv_equals_conv1d(k, d):
    g = torch.Generator().manual_seed(k * d)
    w = torch.randn(32, 16, k, generator=g).double()
    b = torch.randn(32, generator=g, dtype=torch.float64)
    x = torch.randn(2, 16, 13, generator=g, dtype=torch.float64)
    ref = F.conv1d(x, w, b, padding=d * (k - 1) // 2, dilation=d)
    y = ho.packed_conv(x.transpose(1, 2), hifigan.pack_conv(w.float()), b, 32, k, d)
    assert (y.transpose(1, 2) - ref).abs().max().item() < 1e-5


def test_weights_split_into_exact_tf32_halves():
    w = torch.randn(16, 16, 3, generator=torch.Generator().manual_seed(3))
    wp = hifigan.pack_conv(w).reshape(-1, 2, 2)
    hi, lo = wp[:, 0], wp[:, 1]
    assert ((hi.view(torch.int32) & 0x1FFF) == 0).all() and ((lo.view(torch.int32) & 0x1FFF) == 0).all()
    # the packing only permutes: the sorted hi + lo are the sorted weights to 2^-22 relative
    err = ((hi.double() + lo.double()).reshape(-1).sort()[0] - w.double().reshape(-1).sort()[0]).abs() / w.abs().max()
    assert err.max() < 2.0 ** -21


def test_weight_norm_folding_matches_remove_weight_norm():
    gen = _generator(ho.SMALL)
    sd = mk.seeded_state_dict("small")
    gen.load_state_dict(sd, strict=True)
    mods = [gen.conv_pre, gen.ups[0], gen.ups[2], gen.resblocks[4].convs1[2], gen.conv_post]
    folded = [hifigan.folded_weight(m).detach().clone() for m in mods]
    gen.remove_weight_norm()
    for m, f in zip(mods, folded):
        assert not hasattr(m, "weight_g")
        assert torch.equal(m.weight, f) and torch.equal(hifigan.folded_weight(m), f)
    # the ConvTranspose1d norm is per INPUT channel (dim 0 of [C_in, C_out, k])
    v, g = sd["ups.0.weight_v"], sd["ups.0.weight_g"]
    assert g.shape == (v.shape[0], 1, 1)
    assert torch.allclose(folded[1], g * v / v.norm(dim=(1, 2), keepdim=True), rtol=1e-6, atol=0)


@pytest.mark.parametrize("model", ["small", "full"])
def test_both_state_dict_forms_load_strictly(model):
    with open(os.path.join(HERE, "golden", "hifigan_state_dicts.json")) as f:
        trees = json.load(f)
    gen = _generator(mk.MODELS[model]["h"])
    ours = [[k, list(v.shape)] for k, v in gen.state_dict().items()]
    assert ours == trees[model + "_weight_norm"]
    sd = mk.seeded_state_dict(model)
    gen.load_state_dict(sd, strict=True)
    gen.remove_weight_norm()
    assert [[k, list(v.shape)] for k, v in gen.state_dict().items()] == trees[model]
    plain = _generator(mk.MODELS[model]["h"])
    plain.remove_weight_norm()
    plain.load_state_dict(gen.state_dict(), strict=True)                     # a checkpoint saved after removal
    assert torch.equal(plain.resblocks[1].convs2[0].weight, gen.resblocks[1].convs2[0].weight)


@pytest.mark.parametrize("field,value", [
    ("resblock", "2"), ("num_mels", 72), ("upsample_initial_channel", 200), ("upsample_initial_channel", 256),
    ("resblock_kernel_sizes", [3, 6, 11]), ("upsample_kernel_sizes", [16, 16, 4, 4, 5]),
    ("upsample_rates", [8, 8, 2, 2, 3]), ("resblock_dilation_sizes", [[1, 3], [1, 3, 5], [1, 3, 5]])])
def test_unsupported_configurations_raise(field, value):
    with pytest.raises(ValueError, match=field):
        _generator(dict(ho.FULL, **{field: value}))


def test_forward_refuses_cpu_tensors_and_training_under_grad():
    gen = _generator(ho.SMALL)
    with pytest.raises(ValueError, match="CUDA"):
        gen(torch.zeros(1, 128, 2), torch.zeros(1, 2))
    if torch.cuda.is_available():
        gen = gen.cuda().train()
        with pytest.raises(NotImplementedError):
            gen(torch.zeros(1, 128, 2, device="cuda"), torch.zeros(1, 2, device="cuda"))


def test_abi_argument_errors_do_not_touch_the_device():
    from ddsp_svc_b200 import _lib
    lib = _lib.lib()
    p = 16                                     # a non-null, 16-byte aligned address that is never dereferenced
    conv = lambda **kw: lib.b2d_hifigan_conv(*[kw.get(n, d) for n, d in (
        ("x", p), ("sb", 0), ("st", 16), ("sc", 1), ("B", 1), ("T", 8), ("Cin", 16), ("w", p), ("bias", p), ("k", 3),
        ("d", 1), ("N", 16), ("lrelu", 1), ("res", 0), ("acc", 0), ("div", 1.0), ("up", 0), ("src", 0), ("nw", 0),
        ("nb", 0), ("nk", 0), ("ns", 1), ("npad", 0), ("out", p), ("stream", 0))])
    assert conv(x=0) == -1 and conv(src=p) == -1                                   # null x; source without weights
    assert conv(T=0) == -2 and conv(div=0.0) == -2 and conv(up=3, N=32) == -2      # N % up
    assert conv(k=4) == -4 and conv(Cin=24) == -4 and conv(N=40) == -4             # even k, C_in / N % 16
    assert conv(k=11, d=52) == -4                                                  # halo > 256
    assert conv(up=2, N=32, res=p) == -4 and conv(src=p, nw=p, nb=p, nk=2) == -4  # residual with up; source without
    assert conv(st=18) == -3 and conv(x=p + 4) == -3 and conv(out=p + 4) == -3     # unaligned
    assert b"hifigan_conv" in lib.b2d_last_error()
    assert lib.b2d_hifigan_post(0, p, p, 1, 8, 16, p, 0) == -1
    assert lib.b2d_hifigan_post(p, p, p, 1, 0, 16, p, 0) == -2
    assert lib.b2d_hifigan_post(p, p, p, 1, 8, 18, p, 0) == -4
    assert lib.b2d_hifigan_post(p + 4, p, p, 1, 8, 16, p, 0) == -3
