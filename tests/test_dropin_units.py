"""patch_reference(units=True) / unpatch_reference on ddsp.vocoder and encoder.hubert.model (runs where the reference is
importable: DDSP_REFERENCE_ROOT), including a main.py-style Units_Encoder call through the patched reference."""
import pytest
import torch

import ddsp_svc_b200 as pkg
from oracle import ref_loader
from tests import units_oracle as U
from tests.test_oracle_units import _reference_hubert

pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="reference checkout not available (DDSP_REFERENCE_ROOT)")


def test_default_patch_leaves_the_units_encoder_alone():
    V = ref_loader.load()[0]
    orig = V.Units_Encoder
    saved = pkg.patch_reference()
    try:
        assert V.Units_Encoder is orig and "units" not in saved
    finally:
        pkg.unpatch_reference(saved)


def test_units_patch_and_unpatch():
    V = ref_loader.load()[0]
    ref_hubert = _reference_hubert()
    orig = (V.Units_Encoder, V.HubertSoft, ref_hubert.HubertSoft)
    saved = pkg.patch_reference(units=True)
    try:
        assert V.Units_Encoder is pkg.Units_Encoder
        assert V.HubertSoft is pkg.HubertSoft and ref_hubert.HubertSoft is pkg.HubertSoft
    finally:
        pkg.unpatch_reference(saved)
    assert (V.Units_Encoder, V.HubertSoft, ref_hubert.HubertSoft) == orig


def test_main_py_style_contentvec_call_builds_the_package_encoder(tmp_path):
    """main.py's call through the patched reference reaches the package's Units_Encoder and its fairseq loader.  Encoding
    needs a GPU, where the reference is not read: tests/test_gpu_units.py encodes the same checkpoint layout with
    ddsp_svc_b200.Units_Encoder directly."""
    V = ref_loader.load()[0]
    _, fsd = U.fairseq_state_dict(31)
    path = str(tmp_path / "checkpoint_best_legacy_500.pt")
    U.save_fairseq(path, fsd, args=U.fairseq_args())
    saved = pkg.patch_reference(units=True)
    try:
        # main.py: Units_Encoder(args.data.encoder, args.data.encoder_ckpt, args.data.encoder_sample_rate,
        #                        args.data.encoder_hop_size, device=device)
        with pytest.raises(ValueError, match="CUDA device"):
            V.Units_Encoder("contentvec768l12", path, 16000, 320, device="cpu")
        assert V.Units_Encoder is pkg.Units_Encoder
    finally:
        pkg.unpatch_reference(saved)
    model = pkg.load_fairseq_hubert(path)
    assert torch.equal(model.state_dict()["encoder.layers.0.linear1.weight"], fsd["encoder.layers.0.fc1.weight"])
