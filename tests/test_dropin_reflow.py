"""patch_reference(reflow=True) / unpatch_reference on the reference's reflow modules (runs where the reference is
importable: DDSP_REFERENCE_ROOT).  reflow.vocoder needs the enhancer stack's imports (librosa, torchaudio); where they are
missing it is reported under "_not_patched" and the two modules that do import are still patched."""
import sys

import pytest

import ddsp_svc_b200 as pkg
from oracle import ref_loader

pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="reference checkout not available (DDSP_REFERENCE_ROOT)")


def test_default_patch_leaves_the_reflow_modules_alone():
    ref_loader.load()
    import reflow.naive_v2_diff as nv
    import reflow.reflow as rf
    saved = pkg.patch_reference()
    try:
        assert "NaiveV2Diff" not in saved and "RectifiedFlow" not in saved
        assert nv.NaiveV2Diff is not pkg.NaiveV2Diff and rf.RectifiedFlow is not pkg.RectifiedFlow
    finally:
        pkg.unpatch_reference(saved)


def test_reflow_patch_and_unpatch():
    ref_loader.load()
    import reflow.naive_v2_diff as nv
    import reflow.reflow as rf
    orig_nv, orig_rf = nv.NaiveV2Diff, rf.RectifiedFlow
    saved = pkg.patch_reference(reflow=True)
    try:
        assert saved["NaiveV2Diff"] is orig_nv and saved["RectifiedFlow"] is orig_rf
        assert nv.NaiveV2Diff is pkg.NaiveV2Diff and rf.RectifiedFlow is pkg.RectifiedFlow
        rv = sys.modules.get("reflow.vocoder")
        if rv is None:
            assert "reflow.vocoder" in saved["_not_patched"]
        else:                                              # Unit2Wav as load_model_vocoder builds it (reflow/vocoder.py:33-43)
            model = rv.Unit2Wav(44100, 512, 2048, 768, 1, True, 128, 6, 512)
            assert isinstance(model.reflow_model, pkg.RectifiedFlow)
            assert isinstance(model.reflow_model.velocity_fn, pkg.NaiveV2Diff)
    finally:
        pkg.unpatch_reference(saved)
    assert nv.NaiveV2Diff is orig_nv and rf.RectifiedFlow is orig_rf
    rv = sys.modules.get("reflow.vocoder")
    if rv is not None:
        assert rv.NaiveV2Diff is orig_nv and rv.RectifiedFlow is orig_rf
        assert type(rv.Unit2Wav(44100, 512, 2048, 768, 1, True, 128, 6, 512).reflow_model) is orig_rf
