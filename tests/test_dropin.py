"""Drop-in contract: constructor arguments, buffers / state-dict keys and class dispatch match
the reference (SURVEY.md appendix D).  Patching the reference package itself runs only where it is importable
(DDSP_REFERENCE_ROOT)."""
import contextlib
import io
import json
import os
import sys

import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import dropin
from oracle import ref_loader


def test_buffers_and_forward_signature_without_reference():
    import inspect
    m = pkg.Sins(44100, 512, 128, 256, 256, unit2ctrl=pkg.FixedControls())
    assert set(m.state_dict()) == {"sampling_rate", "block_size"}
    assert m.sampling_rate.dtype == torch.int64 and m.sampling_rate.dim() == 0
    sig = inspect.signature(m.forward)
    for name in ("units_frames", "f0_frames", "volume_frames", "spk_id", "spk_mix_dict", "initial_phase", "infer",
                 "max_upsample_dim"):
        assert name in sig.parameters
    c = pkg.CombSub(44100, 512, 256, 512, 256, unit2ctrl=pkg.FixedControls())
    assert set(c.state_dict()) == {"sampling_rate", "block_size"}
    cf = pkg.CombSubFast(44100, 512, unit2ctrl=pkg.FixedControls())
    assert list(cf.state_dict()) == ["sampling_rate", "block_size", "window"] and cf.window.shape == (1024,)
    g = pkg.SineGen(44100, harmonic_num=8)
    assert g.dim == 9 and len(g.state_dict()) == 0
    sm = pkg.SourceModuleHnNSF(44100, harmonic_num=8)
    assert list(sm.state_dict()) == ["l_linear.weight", "l_linear.bias"]
    assert sm.l_linear.weight.shape == (1, 9) and sm.l_sin_gen.dim == 9
    assert "voiced_threshod" in inspect.signature(pkg.SourceModuleHnNSF.__init__).parameters   # reference spelling
    with pytest.raises(ValueError, match="Unknown Model"):
        dropin.build_model(dropin.DotDict({"model": {"type": "Nope"}, "data": {}}))
    # no unit2ctrl argument: the package's own Unit2Control (no dependency on the reference package), same head as the
    # reference's (SURVEY appendix D: dense_out -> 640 outputs for Sins 128/256/256)
    own = pkg.Sins(44100, 512, 128, 256, 256, n_unit=768)
    from ddsp_svc_b200.unit2control import Unit2Control
    assert isinstance(own.unit2ctrl, Unit2Control) and own.unit2ctrl.dense_out.weight_v.shape == (640, 256)
    assert {"unit2ctrl.dense_out.weight_g", "unit2ctrl.dense_out.weight_v", "unit2ctrl.dense_out.bias"} <= set(own.state_dict())
    with pytest.raises(ValueError, match="block_size"):
        pkg.Sins(44100, 441, 128, 256, 256, unit2ctrl=pkg.FixedControls())          # unsupported shapes fail at build time


def test_module_refuses_cpu_tensors():
    m = pkg.Sins(44100, 512, 4, 9, 9, unit2ctrl=pkg.FixedControls())
    with pytest.raises(ValueError, match="CUDA"):
        m(None, torch.zeros(1, 3, 1), None)


def test_state_dict_round_trip_with_the_reference_classes(tmp_path):
    """state-dict keys / shapes of the reference classes: tests/golden/reference_state_dicts.json
    (tests/golden/make_golden_reference.py).  Patching the reference package itself is checked as well when it is
    importable (DDSP_REFERENCE_ROOT)."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_state_dicts.json")) as f:
        ref_sds = json.load(f)
    g = torch.Generator().manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        cases = [("Sins", lambda: pkg.Sins(44100, 512, 128, 256, 256, n_unit=768, n_spk=1)),
                 ("CombSub", lambda: pkg.CombSub(44100, 512, 256, 512, 256, n_unit=768, n_spk=2)),
                 ("CombSubSuperFast", lambda: pkg.CombSubSuperFast(44100, 512, 2048, n_unit=768, n_spk=1)),
                 ("CombSubFast", lambda: pkg.CombSubFast(44100, 512, n_unit=768, n_spk=1)),
                 ("SourceModuleHnNSF", lambda: pkg.SourceModuleHnNSF(44100, harmonic_num=8))]
        saved_sd = None
        for name, make in cases:
            ours = make()
            assert [[k, list(v.shape)] for k, v in ours.state_dict().items()] == ref_sds[name], name
            dtypes = {k: v.dtype for k, v in ours.state_dict().items()}
            sd = {k: (100 * torch.randn(shape, generator=g)).to(dtypes[k]) for k, shape in ref_sds[name]}   # a checkpoint's layout
            ours.load_state_dict(sd)                        # strict, like ddsp/vocoder.py:527
            for k, v in ours.state_dict().items():
                assert torch.equal(v, sd[k]), k
            if name == "CombSubSuperFast":
                saved_sd = sd
        # load_model: config.yaml next to the checkpoint -> class dispatch -> strict load
        import yaml
        cfg = {"data": {"sampling_rate": 44100, "block_size": 512, "encoder_out_channels": 768},
               "model": {"type": "CombSubSuperFast", "win_length": 2048, "n_spk": 1}}
        (tmp_path / "config.yaml").write_text(yaml.safe_dump(cfg))
        torch.save({"global_step": 1, "model": saved_sd}, tmp_path / "model_1.pt")
        model, args = dropin.load_model(str(tmp_path / "model_1.pt"), device="cpu")
        assert isinstance(model, pkg.CombSubSuperFast) and args.model.win_length == 2048
        if not ref_loader.available():
            return
        # patch / unpatch the reference package
        V, _, _ = ref_loader.load()
        saved = pkg.patch_reference()
        try:
            assert V.Sins is pkg.Sins and V.CombSubSuperFast is pkg.CombSubSuperFast
            assert V.CombSubFast is pkg.CombSubFast
            import nsf_hifigan.models as nsf
            assert nsf.SineGen is pkg.SineGen and nsf.SourceModuleHnNSF is pkg.SourceModuleHnNSF
            model2, _ = V.load_model(str(tmp_path / "model_1.pt"), device="cpu")   # the REFERENCE's loader
            assert isinstance(model2, pkg.CombSubSuperFast)
        finally:
            pkg.unpatch_reference(saved)
        assert V.Sins is not pkg.Sins and nsf.SourceModuleHnNSF is not pkg.SourceModuleHnNSF
