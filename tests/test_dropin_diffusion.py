"""patch_reference(diffusion=True) / unpatch_reference on the reference's diffusion modules (runs where the reference is
importable: DDSP_REFERENCE_ROOT), and strict loading of the reference's state dicts into the package's classes.
diffusion.diffusion imports librosa.sequence and diffusion.vocoder the enhancer stack; where they are missing the modules
are reported under "_not_patched" and the ones that do import are still patched."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from oracle import ref_loader

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="reference checkout not available (DDSP_REFERENCE_ROOT)")
MODULES = ("diffusion.vocoder", "diffusion.diffusion", "diffusion.wavenet", "diffusion.naive_v2_diff")
OURS = dict(GaussianDiffusion=pkg.GaussianDiffusion, WaveNet=pkg.WaveNet, NaiveV2Diff=pkg.NaiveV2Diff)


def test_default_patch_leaves_the_diffusion_modules_alone():
    ref_loader.load()
    import diffusion.wavenet as wn
    saved = pkg.patch_reference()
    try:
        assert "diffusion" not in saved and wn.WaveNet is not pkg.WaveNet
    finally:
        pkg.unpatch_reference(saved)


def test_diffusion_patch_and_unpatch():
    ref_loader.load()
    import diffusion.naive_v2_diff as nv
    import diffusion.wavenet as wn
    import reflow.naive_v2_diff as rnv
    orig_wn, orig_nv, orig_rnv = wn.WaveNet, nv.NaiveV2Diff, rnv.NaiveV2Diff
    saved = pkg.patch_reference(diffusion=True)
    try:
        patched = saved["diffusion"]
        assert patched["diffusion.wavenet"]["WaveNet"] is orig_wn and patched["diffusion.naive_v2_diff"]["NaiveV2Diff"] is orig_nv
        assert wn.WaveNet is pkg.WaveNet and nv.NaiveV2Diff is pkg.NaiveV2Diff
        assert rnv.NaiveV2Diff is orig_rnv                                  # the reflow modules stay as they were
        for modname in MODULES:
            mod = sys.modules.get(modname)
            if modname in saved.get("_not_patched", {}):
                continue
            for name in ("GaussianDiffusion", "WaveNet", "NaiveV2Diff"):
                if name in patched[modname]:
                    assert getattr(mod, name) is OURS[name], (modname, name)
        dv = sys.modules.get("diffusion.vocoder")
        if dv is None:
            assert "diffusion.vocoder" in saved["_not_patched"] and "diffusion.diffusion" in saved["_not_patched"]
        else:                                                  # Unit2Wav as diffusion/vocoder.py:221-235 builds it
            model = dv.Unit2Wav(44100, 512, 768, 1, True, 128, 20, 512)
            assert isinstance(model.diff_model, pkg.GaussianDiffusion) and isinstance(model.diff_model.denoise_fn, pkg.WaveNet)
        # a reference WaveNet's parameters load strictly into the patched class
        ref = orig_wn(128, 2, 64, 256)
        ours = wn.WaveNet(128, 2, 64, 256)
        ours.load_state_dict(ref.state_dict(), strict=True)
        assert torch.equal(ours.residual_layers[1].dilated_conv.weight, ref.residual_layers[1].dilated_conv.weight)
    finally:
        pkg.unpatch_reference(saved)
    assert wn.WaveNet is orig_wn and nv.NaiveV2Diff is orig_nv and rnv.NaiveV2Diff is orig_rnv


@pytest.mark.parametrize("key,make", [
    ("Unit2Wav.diff_model", lambda: pkg.GaussianDiffusion(pkg.WaveNet(128, 20, 512, 256), out_dims=128)),
    ("Unit2WavFast.diff_model", lambda: pkg.GaussianDiffusion(
        pkg.NaiveV2Diff(mel_channels=128, dim=512, num_layers=6, condition_dim=128, use_mlp=False), out_dims=128))])
def test_a_checkpoints_diffusion_state_dict_loads_strictly(key, make):
    """a state dict with the reference's keys, shapes and buffer values (tests/golden/diffusion_state_dicts.json,
    diffusion_buffers.npz) -- what a DiffusionNew / DiffusionFast model_*.pt holds under diff_model."""
    with open(os.path.join(HERE, "golden", "diffusion_state_dicts.json")) as f:
        shapes = json.load(f)[key]
    bufs = np.load(os.path.join(HERE, "golden", "diffusion_buffers.npz"))
    g = torch.Generator().manual_seed(1)
    sd = {k: torch.from_numpy(bufs[k]).float().reshape(s) if k in bufs else torch.randn(s, generator=g) for k, s in shapes}
    model = make()
    model.load_state_dict(sd, strict=True)
    assert torch.equal(model.alphas_cumprod, sd["alphas_cumprod"])
