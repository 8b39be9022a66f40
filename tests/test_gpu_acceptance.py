"""Acceptance run on the GPU: the reference's OWN call (main.py:259, `model(seg_units, seg_f0, seg_volume, spk_id=...,
spk_mix_dict=...)` under torch.no_grad, then `seg_output *= mask` in place, main.py:260) through this package's
synthesizers AND its Unit2Control, built by `load_model` from a checkpoint + config.yaml (the drop-in of the reference's
loader), against the reference classes' waveforms for the same checkpoint and inputs -- real torch.split views of
dense_out, real spk_id embedding / spk_mix_dict.

The reference side is stored in tests/golden/acceptance_*.npz (tests/golden/make_golden_reference.py: the reference
classes on the CPU in fp32, with this package's seeded initial weights loaded strictly, and the white noise they drew).
The recorded noise is fed to this package's module (`noise=`), so the full signal is comparable; the exact main.py call
without `noise=` (in-kernel Philox) is checked on its deterministic part and on the noise level."""
import io
import contextlib

import numpy as np
import pytest
import torch
import yaml

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import dropin
from tests import report, util
from tests.golden import cases as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P, NU = 44100, 512, 768
NF = 80                                             # one short main.py segment (~0.9 s), B = 1
GATE_RMS = 1e-4                                     # the north star's bound; 1e-8-level parity is pinned by the golden tests


CASES = {
    "Sins": dict(model={"type": "Sins", "n_harmonics": 128, "n_mag_allpass": 256, "n_mag_noise": 256, "n_spk": 2},
                 make=lambda M: M.Sins(SR, P, 128, 256, 256, n_unit=NU, n_spk=2), uniform=True, parts=True),
    "CombSub": dict(model={"type": "CombSub", "n_mag_allpass": 256, "n_mag_harmonic": 512, "n_mag_noise": 256, "n_spk": 2},
                    make=lambda M: M.CombSub(SR, P, 256, 512, 256, n_unit=NU, n_spk=2), uniform=True, parts=True),
    "CombSubSuperFast": dict(model={"type": "CombSubSuperFast", "win_length": 2048, "n_spk": 2},
                             make=lambda M: M.CombSubSuperFast(SR, P, 2048, n_unit=NU, n_spk=2), uniform=False, parts=False),
    "CombSubFast": dict(model={"type": "CombSubFast", "n_spk": 2},
                        make=lambda M: M.CombSubFast(SR, P, n_unit=NU, n_spk=2), uniform=True, parts=False),
}


def seeded_state_dict(kind):
    """the checkpoint of both sides: this package's initial weights under a fixed seed (CPU RNG)"""
    with contextlib.redirect_stdout(io.StringIO()):
        torch.manual_seed(1)
        return CASES[kind]["make"](pkg).state_dict()


def inputs():
    g = torch.Generator().manual_seed(2)
    units = torch.randn(1, NF, NU, generator=g)
    f0 = 220.0 * 2 ** (torch.rand(1, NF, 1, generator=g) * 0.3)
    f0[:, 40:48] = 0.0                              # an unvoiced stretch, as f0 extractors produce
    volume = 0.1 * torch.rand(1, NF, 1, generator=g)
    mask = (torch.rand(1, NF * P, generator=g) > 0.1).float()
    return units, f0, volume, mask


def calls():
    spk_id = torch.LongTensor([[2]])
    return [dict(spk_id=spk_id, spk_mix_dict=None), dict(spk_id=spk_id, spk_mix_dict={1: 0.3, 2: 0.7})]


def source_module_inputs():
    g = torch.Generator().manual_seed(4)
    f0 = 200.0 + 50.0 * torch.rand(2, 20, generator=g)
    f0[:, 5:8] = 0.0
    return f0, 512


@pytest.mark.parametrize("kind", list(CASES))
def test_main_py_call_reference_vs_patched(kind, tmp_path):
    case = CASES[kind]
    cfg = {"data": {"sampling_rate": SR, "block_size": P, "encoder_out_channels": NU}, "model": case["model"]}
    (tmp_path / "config.yaml").write_text(yaml.safe_dump(cfg))
    torch.save({"global_step": 1, "model": seeded_state_dict(kind)}, tmp_path / "model_1.pt")
    with contextlib.redirect_stdout(io.StringIO()):
        model, args = dropin.load_model(str(tmp_path / "model_1.pt"), device=DEV)
    assert isinstance(model, getattr(pkg, kind))
    units, f0, volume, mask = (t.to(DEV) for t in inputs())
    with torch.no_grad():
        for i, kw in enumerate(calls()):
            gold = np.load(G.path("acceptance_%s_%d" % (kind, i)))
            r_sig, r_hid = torch.from_numpy(gold["signal"]), torch.from_numpy(gold["hidden"])
            noise = torch.from_numpy(gold["noise"]).to(DEV)
            kw = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()}
            # (1) same noise samples -> the whole signal is comparable
            sig, hidden, (s_h, s_n) = model(units, f0, volume, noise=noise, **kw)
            # this package's Unit2Control (fused kernels + fp32 library GEMMs) against the reference's class in fp32
            assert util.rms(hidden.cpu() - r_hid) < 1e-4 * max(util.rms(r_hid), 1e-6)
            e = util.rms(sig.cpu() - r_sig)
            report.record("acceptance/%s/%s" % (kind, "mix" if kw["spk_mix_dict"] else "spk"), err=e,
                          max=(sig.cpu() - r_sig).abs().max().item(), signal_rms=util.rms(r_sig))
            assert e < GATE_RMS
            if case["parts"]:
                r_h = torch.from_numpy(gold["harmonic"])
                r_n = r_sig - r_h                   # the reference's signal is harmonic + noise
                assert util.rms(s_h.cpu() - r_h) < GATE_RMS and util.rms(s_n.cpu() - r_n) < GATE_RMS
            # (2) the exact main.py lines: no `noise=`, then the in-place mask multiply on the returned tensor
            seg_output, _, (s_h2, s_n2) = model(units, f0, volume, **kw)
            if case["parts"]:
                assert util.rms(s_h2.cpu() - r_h) < GATE_RMS                               # deterministic part
                lvl = util.rms(s_n2.cpu()) / max(util.rms(r_n), 1e-12)
                assert 0.9 < lvl < 1.1                                                 # same noise level, other samples
                keep_h = s_h2.clone()
            else:
                lvl = util.rms(seg_output.cpu()) / max(util.rms(r_sig), 1e-12)
                assert 0.8 < lvl < 1.25
            before = seg_output.clone()
            seg_output *= mask                                                          # main.py:260
            assert torch.equal(seg_output, before * mask)
            if case["parts"]:
                assert torch.equal(s_h2, keep_h)                                       # outputs are not aliased


def test_enhancer_source_module_through_patch_reference():
    """enhancer.py's generator builds `SourceModuleHnNSF(...)`; this package's fused module with the reference class's
    state dict (this package's seeded initial weights) and the reference's random phases / noise fed in gives the
    reference's output (tests/golden/acceptance_source_module.npz)."""
    gold = np.load(G.path("acceptance_source_module"))
    torch.manual_seed(3)
    ours = pkg.SourceModuleHnNSF(SR, harmonic_num=8).to(DEV).eval()
    f0, upp = source_module_inputs()
    rand_ini = torch.from_numpy(gold["rand_ini"]).to(DEV)
    with torch.no_grad():
        out = ours(f0.to(DEV), upp, rand_ini=rand_ini, noise=torch.from_numpy(gold["noise"]).to(DEV))
    ref_out = torch.from_numpy(gold["out"])
    e = util.rms(out.cpu() - ref_out)
    report.record("acceptance/source_module", err=e, rms=util.rms(ref_out))
    assert out.shape == ref_out.shape and e < 1e-4
