"""patch_reference(enhancer=True) / unpatch_reference on the reference's enhancer module (runs where the reference is
importable: DDSP_REFERENCE_ROOT).  The enhancer itself runs on the GPU in tests/test_gpu_realtime.py."""
import sys

import pytest

import ddsp_svc_b200 as pkg
from ddsp_svc_b200.enhancer import Enhancer
from oracle import ref_loader

pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="reference checkout not available (DDSP_REFERENCE_ROOT)")


def test_default_patch_leaves_the_enhancer_alone():
    ref_loader.load()
    saved = pkg.patch_reference()
    try:
        mod = sys.modules.get("enhancer")
        assert mod is None or mod.Enhancer is not Enhancer
        assert "enhancer" not in saved
    finally:
        pkg.unpatch_reference(saved)


def test_enhancer_patch_and_unpatch():
    ref_loader.load()
    saved = pkg.patch_reference(enhancer=True)
    try:
        if "enhancer" in saved.get("_not_patched", {}):
            pytest.skip("the reference's enhancer module does not import here: %s" % saved["_not_patched"]["enhancer"])
        import enhancer as ref_enhancer
        original = saved["enhancer"]["enhancer"]["Enhancer"]
        assert ref_enhancer.Enhancer is Enhancer and original is not Enhancer
    finally:
        pkg.unpatch_reference(saved)
    assert ref_enhancer.Enhancer is original
