"""GPU parity of this package's Unit2Control (fused kernels of csrc/unit2control.cu + library GEMMs) against the reference's
own class (ddsp/unit2control.py with PCmer / ConformerNaiveEncoder) evaluated on the CPU in fp32, on the same weights
(this package's seeded initialisation, loaded strictly into the reference class) and inputs.  The reference's outputs are
stored under tests/golden/ (u2c_gpu_*.npz, u2c_sins_e2e.npz: tests/golden/make_golden_reference.py) as a fixed seeded
sample of their elements."""
import json

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200.unit2control import Unit2Control
from tests import report, util
from tests.golden import cases as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

VARIANTS = {
    "pcmer_sins": (dict(), {"amplitudes": 128, "group_delay": 256, "noise_magnitude": 256}),
    "pcmer_sins_fused_attention": (dict(), {"amplitudes": 128, "group_delay": 256, "noise_magnitude": 256}),
    "naive_superfast": (dict(use_naive_v2=True, use_conv_stack=True, use_pitch_aug=True),
                        {"harmonic_magnitude": 1025, "harmonic_phase": 1025, "noise_magnitude": 1025, "noise_phase": 1025}),
    "pcmer_norm_plainconv": (dict(pcmer_norm=True, use_conv_stack=False), {"a": 33, "b": 7}),
}


def calls_of(kw):
    calls = [dict(spk_id=torch.LongTensor([[2], [3]])), dict(spk_id=torch.LongTensor([[1]]), spk_mix_dict={1: 0.25, 3: 0.75})]
    if kw.get("use_pitch_aug"):
        calls.append(dict(spk_id=torch.LongTensor([[1], [1]]), aug_shift=torch.tensor([[[2.0]], [[-3.0]]])))
    return calls


def _sample(n, seed, k=16384):
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:k].sort().values


def _inputs(B, T, n_unit, seed):
    g = torch.Generator().manual_seed(seed)
    units = torch.randn(B, T, n_unit, generator=g)
    f0 = 220.0 * 2 ** (torch.rand(B, T, 1, generator=g) * 2 - 1)
    f0[:, 5:9] = 0.0
    phase = (torch.rand(B, T, 1, generator=g) * 2 - 1) * 3.14159
    volume = 0.2 * torch.rand(B, T, 1, generator=g)
    return units, f0, phase, volume


@pytest.mark.parametrize("name", list(VARIANTS))
def test_unit2control_matches_the_reference_class(name):
    kw, splits = VARIANTS[name]
    gold = np.load(G.path("u2c_gpu_" + name.replace("_fused_attention", "")))
    torch.manual_seed(3)
    ours = Unit2Control(768, 3, splits, **kw)
    assert [[k, list(v.shape)] for k, v in ours.state_dict().items()] == json.loads(str(gold["keys_shapes"]))
    ours = ours.to(DEV).eval()
    ours.fused_attention = name.endswith("fused_attention")      # the opt-in one-kernel linear attention (csrc/linear_attention.cu)
    B, T = 2, 150
    units, f0, phase, volume = _inputs(B, T, 768, 4)
    for i, c in enumerate(calls_of(kw)):
        cg = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in c.items()}
        with torch.no_grad():
            got_c, got_h = ours(units.to(DEV), f0.to(DEV), phase.to(DEV), volume.to(DEV), **cg)
        assert list(got_c.keys()) == list(splits.keys())
        first = next(iter(got_c.values()))
        assert first.stride(1) == sum(splits.values())                      # views of one dense tensor, like torch.split
        dense_g = torch.cat([got_c[k].cpu() for k in got_c], -1).reshape(-1)
        hid_g = got_h.cpu().reshape(-1)
        dense_g, hid_g = dense_g[_sample(dense_g.numel(), 100 + i)], hid_g[_sample(hid_g.numel(), 200 + i)]
        dense_w, hid_w = torch.from_numpy(gold["controls_%d" % i]), torch.from_numpy(gold["hidden_%d" % i])
        e_c = util.rms(dense_g - dense_w) / max(util.rms(dense_w), 1e-12)
        e_h = util.rms(hid_g - hid_w) / max(util.rms(hid_w), 1e-12)
        report.record("unit2control/%s/%d" % (name, i), controls_rel_rms=e_c, hidden_rel_rms=e_h,
                      controls_max=(dense_g - dense_w).abs().max().item())
        assert e_c < 2e-5 and e_h < 2e-5


def test_sins_forward_end_to_end_without_the_reference_unit2ctrl():
    """Sins built WITHOUT a unit2ctrl argument owns this package's Unit2Control: with the same weights and the noise the
    reference drew, the whole forward (control network + DSP) matches the reference's CPU forward within the north-star
    bound."""
    gold = np.load(G.path("u2c_sins_e2e"))
    torch.manual_seed(5)
    ours = pkg.Sins(44100, 512, 128, 256, 256, n_unit=768, n_spk=2)
    assert isinstance(ours.unit2ctrl, Unit2Control)
    ours = ours.to(DEV).eval()
    units, f0, _, volume = _inputs(1, 90, 768, 6)
    spk = torch.LongTensor([[2]])
    want, noise = torch.from_numpy(gold["signal"]), torch.from_numpy(gold["noise"])
    with torch.no_grad():
        got, got_h, (gh, gn) = ours(units.to(DEV), f0.to(DEV), volume.to(DEV), spk_id=spk.to(DEV), noise=noise.to(DEV))
    e = util.rms(got.cpu() - want)
    report.record("unit2control/sins_e2e", err=e, signal_rms=util.rms(want))
    assert e < 1e-4 and e < 2e-3 * util.rms(want)
