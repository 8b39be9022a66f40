"""patch_reference(hifigan=True) / unpatch_reference on nsf_hifigan.models (runs where the reference is importable:
DDSP_REFERENCE_ROOT): load_model then builds the package's Generator from a checkpoint and its config.json, and the
default patch leaves the reference's class alone."""
import json
import os
import warnings

import pytest
import torch

import ddsp_svc_b200 as pkg
from oracle import ref_loader
from tests import hifigan_oracle as ho
from tests.golden import make_golden_hifigan as mk

pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="reference checkout not available (DDSP_REFERENCE_ROOT)")


def test_default_patch_leaves_the_generator_alone():
    ref_loader.load()
    import nsf_hifigan.models as m
    orig = m.Generator
    saved = pkg.patch_reference()
    try:
        assert "Generator" not in saved and m.Generator is orig
    finally:
        pkg.unpatch_reference(saved)
    assert m.Generator is orig


def test_hifigan_patch_load_model_and_unpatch(tmp_path):
    ref_loader.load()
    import nsf_hifigan.models as m
    orig = m.Generator
    with open(os.path.join(tmp_path, "config.json"), "w") as f:
        json.dump(ho.SMALL, f)
    ckpt = os.path.join(tmp_path, "model.ckpt")
    torch.save({"generator": mk.seeded_state_dict("small")}, ckpt)
    saved = pkg.patch_reference(hifigan=True)
    try:
        assert saved["Generator"] is orig and m.Generator is pkg.Generator
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            gen, h = m.load_model(ckpt, device="cpu")          # strict load, eval(), remove_weight_norm()
        assert type(gen) is pkg.Generator and not gen.training
        assert not hasattr(gen.conv_pre, "weight_g")
    finally:
        pkg.unpatch_reference(saved)
    assert m.Generator is orig
    ref = orig(h)                       # after unpatching: the reference's __init__ calls super(Generator, self)
    ref.load_state_dict(mk.seeded_state_dict("small"), strict=True)
    ref.remove_weight_norm()
    assert torch.equal(gen.ups[1].weight, ref.ups[1].weight)
