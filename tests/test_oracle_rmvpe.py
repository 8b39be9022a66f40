"""Host side of the RMVPE drop-in (ddsp_svc_b200.rmvpe), no GPU: the resample table against torchaudio, the HTK mel
basis against torchaudio's melscale_fbanks, BatchNorm folding and the ConvTranspose2d polyphase rewrite against
F.conv2d / F.conv_transpose2d in float64, the parameter tree, fp16 checkpoints, configuration errors, the float64
oracle against the live reference (where it is importable) and patch_reference(rmvpe=True) through F0_Extractor."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import mel as M, rmvpe as R
from oracle import ref_loader
from tests import rmvpe_oracle as ro
from tests.golden import make_golden_rmvpe as mk


@pytest.mark.parametrize("sr", [22050, 32000, 44100, 48000, 8000, 11025])
def test_resample_table_matches_torchaudio(sr):
    import torchaudio
    ref = torchaudio.transforms.Resample(sr, 16000, lowpass_filter_width=128)
    table, width, orig, new = R.resample_table(sr)
    assert width == ref.width and (new, table.shape[1]) == tuple(ref.kernel.shape[::2])
    assert torch.equal(table, ref.kernel[:, 0])


@pytest.mark.parametrize("n,sr", [(1412, 44100), (88200, 44100), (1000, 22050), (48001, 48000)])
def test_resample_length_and_oracle(n, sr):
    import torchaudio
    x = torch.randn(2, n, generator=torch.Generator().manual_seed(n), dtype=torch.float64)
    ref = torchaudio.transforms.Resample(sr, 16000, lowpass_filter_width=128).double()(x)
    assert R.resampled_length(n, sr) == ref.shape[1]
    assert (ro.resample(x, sr) - ref).abs().max() < 1e-6


def test_resampled_length_examples():
    assert R.resampled_length(1412, 44100) == 513 and R.resampled_length(88200, 44100) == 32000


def test_htk_mel_basis():
    import torchaudio
    basis = R.mel_basis()
    ref = torchaudio.functional.melscale_fbanks(513, 30.0, 8000.0, 128, 16000, norm="slaney", mel_scale="htk").T
    assert basis.shape == (128, 513) and basis.dtype == np.float32
    assert np.abs(basis - ref.numpy()).max() < 1e-5 * np.abs(basis).max()        # torchaudio works in fp32
    lohi = M._support(basis)
    assert (lohi[:, 1] - lohi[:, 0] >= 2).all() and (lohi[:, 1] - lohi[:, 0] <= 21).all()
    # the Slaney basis is unchanged by the htk switch
    assert np.array_equal(M.mel_filterbank(44100, 2048, 128, 40, 16000), M.mel_filterbank(44100, 2048, 128, 40, 16000,
                                                                                        htk=False))


def test_bn_fold():
    torch.manual_seed(0)
    conv, bn = torch.nn.Conv2d(8, 12, 3, padding=1, bias=False).double(), torch.nn.BatchNorm2d(12).double()
    with torch.no_grad():
        bn.running_mean.uniform_(-1, 1); bn.running_var.uniform_(0.5, 2); bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-1, 1)
    bn.eval()
    x = torch.randn(2, 8, 10, 16, dtype=torch.float64)
    w, b = R.fold_bn(conv.weight, bn)
    assert torch.allclose(F.conv2d(x, w, b, padding=1), bn(conv(x)), atol=1e-12)


@pytest.mark.parametrize("T,Fq", [(1, 1), (3, 4), (8, 16)])
def test_polyphase2d(T, Fq):
    g = torch.Generator().manual_seed(T)
    x = torch.randn(2, 6, T, Fq, generator=g, dtype=torch.float64)
    w = torch.randn(6, 5, 3, 3, generator=g, dtype=torch.float64)
    ref = F.conv_transpose2d(x, w, stride=2, padding=1, output_padding=1)          # [2, 5, 2T, 2F]
    y = F.conv2d(F.pad(x, (0, 1, 0, 1)), R.polyphase2d(w))                           # [2, 4 C_out, T, F]
    y = y.view(2, 2, 2, 5, T, Fq).permute(0, 3, 4, 1, 5, 2).reshape(2, 5, 2 * T, 2 * Fq)
    assert torch.allclose(y, ref, atol=1e-12)


def test_parameter_tree_and_counts():
    m = R.E2E0(4, 1, (2, 2))
    n = sum(p.numel() for p in m.parameters())
    tf = sum(p.numel() for k, p in m.named_parameters() if k.startswith("unet.tf."))
    assert round(n / 1e6, 1) == 92.0 and round(tf / 1e6, 2) == 1.57
    keys = set(m.state_dict())
    for k in ("unet.encoder.bn.running_var", "unet.encoder.layers.0.conv.0.shortcut.weight",
              "unet.decoder.layers.4.conv1.0.weight", "unet.decoder.layers.0.conv2.0.shortcut.bias",
              "unet.intermediate.layers.3.conv.3.conv.4.num_batches_tracked", "fc.0.gru.weight_hh_l0_reverse",
              "fc.1.weight", "cnn.bias", "unet.tf.layers.4.conv.0.weight"):
        assert k in keys, k


def test_fp16_checkpoint_loads(tmp_path):
    torch.manual_seed(1)
    src = R.E2E0(1, 1, (2, 2), en_de_layers=2, inter_layers=1)
    sd = {k: (v.half() if v.is_floating_point() else v) for k, v in src.state_dict().items()}
    path = tmp_path / "model.pt"
    torch.save({"model": sd}, path)
    dst = R.E2E0(1, 1, (2, 2), en_de_layers=2, inter_layers=1)
    dst.load_state_dict(torch.load(path)["model"], strict=True)
    assert dst.fc[1].weight.dtype == torch.float32
    assert torch.equal(dst.fc[1].weight, src.fc[1].weight.half().float())


def test_rmvpe_loads_fp16_full_checkpoint(tmp_path):
    sd = {k: (v.half() if v.is_floating_point() else v) for k, v in R.E2E0(4, 1, (2, 2)).state_dict().items()}
    torch.save({"model": sd}, tmp_path / "model.pt")
    ex = R.RMVPE(str(tmp_path / "model.pt"))
    assert not ex.model.training and ex.model.cnn.weight.dtype == torch.float32
    assert torch.equal(ex.model.cnn.weight, sd["cnn.weight"].float())


@pytest.mark.parametrize("kw,field", [(dict(n_gru=2), "n_gru"), (dict(n_gru=0), "n_gru"),
                                      (dict(kernel_size=(1, 2)), "kernel_size"), (dict(in_channels=2), "in_channels"),
                                      (dict(en_out_channels=8), "en_out_channels"), (dict(n_blocks=0), "n_blocks"),
                                      (dict(en_de_layers=8), "en_de_layers"), (dict(inter_layers=0), "inter_layers")])
def test_configuration_errors(kw, field):
    args = dict(n_blocks=1, n_gru=1, kernel_size=(2, 2), en_de_layers=2, inter_layers=1)
    args.update(kw)
    with pytest.raises(ValueError, match=field):
        R.E2E0(**args)


def test_cpu_inputs_raise(tmp_path):
    m = R.E2E0(1, 1, (2, 2), en_de_layers=2, inter_layers=1).eval()
    with pytest.raises(ValueError, match="CUDA"):
        m(torch.zeros(1, 128, 32))
    torch.save({"model": {}}, tmp_path / "model.pt")
    ex = R.RMVPE(str(tmp_path / "model.pt"))
    with pytest.raises(ValueError, match="CUDA"):
        ex.infer_from_audio(np.zeros(2000, np.float32), 16000, device="cpu")
    with pytest.raises(ValueError, match="CUDA"):
        ex.infer_batch(torch.zeros(1, 2000), 16000)
    with pytest.raises(NotImplementedError, match="librosa"):
        ex.infer_from_audio(np.zeros(2000, np.float32), 16000, use_viterbi=True)


# ---- against the live reference (DDSP_REFERENCE_ROOT) -----------------------------------------------------------------
def _reference_rmvpe():
    """the reference's encoder.rmvpe, importable without librosa, with spec.py given an HTK basis that does not come
    from the package under test (tests/golden/make_golden_rmvpe.reference)"""
    return mk.reference()


needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="reference checkout not available "
                                                                  "(DDSP_REFERENCE_ROOT)")


@needs_ref
def test_state_dict_matches_reference_tree():
    rm = _reference_rmvpe()
    for args in ((4, 1, (2, 2)), (1, 1, (2, 2), 2, 1)):
        ref = rm.E2E0(*args)
        ours = R.E2E0(*args)
        assert {k: tuple(v.shape) for k, v in ref.state_dict().items()} == \
               {k: tuple(v.shape) for k, v in ours.state_dict().items()}
        ours.load_state_dict(ref.state_dict(), strict=True)


@needs_ref
def test_oracle_against_reference():
    rm = _reference_rmvpe()
    from encoder.rmvpe.utils import to_local_average_f0
    m = ro.seeded_model(n_blocks=1, en_de_layers=2, inter_layers=1)
    ref = rm.E2E0(1, 1, (2, 2), en_de_layers=2, inter_layers=1)
    ref.load_state_dict(m.state_dict(), strict=True)
    ref.eval().double()
    g = torch.Generator().manual_seed(3)
    audio = 0.3 * torch.randn(1, 44100 // 4 + 17, generator=g, dtype=torch.float64)
    with torch.no_grad():
        import torchaudio
        a16 = torchaudio.transforms.Resample(44100, 16000, lowpass_filter_width=128).double()(audio)
        mel_ref = rm.MelSpectrogram(128, 16000, 1024, 160, None, 30, 8000).double()(a16, center=True)
        assert (ro.log_mel(ro.resample(audio, 44100)) - mel_ref).abs().max() < 1e-5
        n = mel_ref.shape[-1]
        hid_ref = ref(F.pad(mel_ref, (0, 32 * ((n - 1) // 32 + 1) - n)))[:, :n]
        hid = ro.mel2hidden(m, mel_ref)
        assert (hid - hid_ref).abs().max() < 1e-9
        f0_ref = to_local_average_f0(hid_ref.float(), thred=0.03)
        assert np.allclose(ro.decode(hid_ref.float())[0].numpy(), f0_ref, rtol=1e-6)


@needs_ref
def test_decode_oracle_against_reference_constructed():
    _reference_rmvpe()
    from encoder.rmvpe.utils import to_local_average_f0
    s = ro.constructed_saliences()[None]
    assert np.array_equal(ro.decode(s)[0].numpy(), to_local_average_f0(s, thred=0.03))


@needs_ref
def test_patch_through_f0_extractor(tmp_path, monkeypatch):
    _reference_rmvpe()
    import ddsp.vocoder as V
    import encoder.rmvpe as rm
    import encoder.rmvpe.inference as ri
    import encoder.rmvpe.model as rmod
    orig = (rm.RMVPE, ri.RMVPE, rmod.E2E0)
    os.makedirs(tmp_path / "pretrain" / "rmvpe")
    torch.save({"model": {}}, tmp_path / "pretrain" / "rmvpe" / "model.pt")
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(V, "F0_KERNEL", {})
    saved = pkg.patch_reference()
    try:
        assert "rmvpe" not in saved and rm.RMVPE is orig[0]
    finally:
        pkg.unpatch_reference(saved)
    saved = pkg.patch_reference(rmvpe=True)
    try:
        assert rm.RMVPE is pkg.RMVPE and ri.RMVPE is pkg.RMVPE and rmod.E2E0 is pkg.E2E0 and ri.E2E0 is pkg.E2E0
        ext = V.F0_Extractor("rmvpe", 44100, 512)
        assert type(ext.rmvpe) is pkg.RMVPE and type(ext.rmvpe.model) is pkg.E2E0
    finally:
        pkg.unpatch_reference(saved)
    assert (rm.RMVPE, ri.RMVPE, rmod.E2E0) == orig


@needs_ref
def test_patch_reports_a_cached_reference_instance(monkeypatch):
    _reference_rmvpe()
    import ddsp.vocoder as V
    import encoder.rmvpe as rm
    monkeypatch.setattr(V, "F0_KERNEL", {"rmvpe": object.__new__(rm.RMVPE)})
    saved = pkg.patch_reference(rmvpe=True)
    try:
        assert "ddsp.vocoder.F0_KERNEL['rmvpe']" in saved["_not_patched"]
    finally:
        pkg.unpatch_reference(saved)
