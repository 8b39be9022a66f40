"""The key-shifted mel on the GPU (csrc/mel.cu's mel_keyshift_kernel through mel.STFT.get_mel_keyshift) against the
reference's fixtures (tests/golden/keyshift_mel_*.npz) and a float64 restatement at preprocess.py's sizes, its
determinism and refusals, and the drop-in Vocoder (extract with resampling and a shift, infer on the package's
generator against the hifigan_small_* goldens)."""
import functools
import json
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import mel as pm
from ddsp_svc_b200 import rmvpe
from oracle import mel as om
from tests import hifigan_oracle as ho
from tests.keyshift_mel_oracle import mel64
from tests import report
from tests.golden import make_golden_hifigan as mk
from tests.golden import make_golden_keyshift_mel as GK

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL_MAX, TOL_RMS = 2e-3, 5e-5          # the keyshift-0 kernel's bounds in log-mel (tests/test_gpu_mel.py)
RATIO = 3.0                            # kernel error <= RATIO x the fp32 reference's own error against float64


def _stft(hop=512):
    return pm.STFT(44100, 128, 2048, 2048, hop, 40, 16000)


@pytest.mark.parametrize("name", list(GK.CASES))
def test_keyshift_mel_matches_reference_fixture(name):
    z = np.load(GK.path(name))
    got = _stft(int(z["hop"])).get_mel_keyshift(torch.from_numpy(z["y"]).to(DEV), float(z["keyshift"])).cpu().numpy()
    assert got.shape == z["mel"].shape
    d = got.astype(np.float64) - z["mel"]
    report.record("keyshift_mel/" + name, max=float(np.abs(d).max()), rms=float(np.sqrt((d ** 2).mean())))
    assert np.abs(d).max() < TOL_MAX and np.sqrt((d ** 2).mean()) < TOL_RMS


@pytest.mark.parametrize("keyshift", [-5.0, 4.98])
def test_batch_of_ten_second_clips_against_float64(keyshift):
    """16 x 10 s, sampled rows: the kernel's error against float64 stays within RATIO x the fp32 reference's"""
    B, T = 16, 441000
    g = torch.Generator().manual_seed(21)
    y = 0.1 * torch.randn(B, T, generator=g)
    a = _stft().get_mel_keyshift(y.to(DEV), keyshift)
    assert torch.isfinite(a).all()
    for r in (0, 11):
        ref = mel64(y[r:r + 1], 512, keyshift)
        with torch.no_grad():
            ref32 = om.get_mel(y[r:r + 1], keyshift=keyshift).double()
        d, d32 = a[r:r + 1].cpu().double() - ref, ref32 - ref
        e, e32 = d.pow(2).mean().sqrt().item(), d32.pow(2).mean().sqrt().item()
        report.record("keyshift_mel/b16_row%d_ks%g" % (r, keyshift), max=d.abs().max().item(), rms=e, ref32_rms=e32)
        assert e <= RATIO * e32 and d.abs().max().item() < TOL_MAX, (e, e32)


def test_two_calls_are_bit_identical_and_an_unshifted_length_is_get_mel():
    g = torch.Generator().manual_seed(22)
    y = (0.1 * torch.randn(3, 512 * 40 + 17, generator=g)).to(DEV)
    st = _stft()
    a = st.get_mel_keyshift(y, 2.7)
    assert torch.equal(a, st.get_mel_keyshift(y, 2.7))
    assert pm.keyshift_n_fft(2048, 0.001) == 2048
    assert torch.equal(st.get_mel_keyshift(y, 0.001), st.get_mel(y))
    assert torch.equal(st.get_mel_keyshift(y, 0), st.get_mel(y))


def test_range_grad_and_cpu_refusals():
    st = _stft()
    y = torch.zeros(1, 8192, device=DEV)
    with pytest.raises(NotImplementedError, match="keyshift in about"):
        st.get_mel_keyshift(y, 7.1)
    with pytest.raises(NotImplementedError, match="keyshift in about"):
        st.get_mel_keyshift(y, -30.0)
    with pytest.raises(NotImplementedError, match="no backward"):
        st.get_mel_keyshift(y.clone().requires_grad_(), -5.0)
    with torch.no_grad():
        assert st.get_mel_keyshift(y.clone().requires_grad_(), -5.0).shape[1] == 128
    with pytest.raises(ValueError, match="CUDA"):
        st.get_mel_keyshift(y.cpu(), -5.0)
    with pytest.raises(NotImplementedError):
        st.get_mel(y, keyshift=2)                               # get_mel itself keeps covering keyshift 0 only


def _write_vocoder(tmp_path, h):
    cfg = dict(ho.SMALL, sampling_rate=44100, num_mels=128, n_fft=2048, win_size=2048, hop_size=512, fmin=40,
               fmax=16000)
    cfg.update(h)
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    ckpt = tmp_path / "model.ckpt"
    torch.save({"generator": mk.seeded_state_dict("small")}, str(ckpt))
    return str(ckpt)


def test_vocoder_extract_resamples_and_shifts(tmp_path):
    voc = pkg.Vocoder("nsf-hifigan", _write_vocoder(tmp_path, {}), device=DEV)
    assert (voc.vocoder_sample_rate, voc.vocoder_hop_size, voc.dimension) == (44100, 512, 128)
    g = torch.Generator().manual_seed(23)
    y48 = 0.1 * torch.randn(1, 48000 * 2, generator=g)
    k, width, orig, new = rmvpe.resample_table(48000, 44100)
    x = F.pad(y48.double(), (width, width + orig))
    y44 = F.conv1d(x[:, None], k.double()[:, None], stride=orig).transpose(1, 2).reshape(1, -1)
    y44 = y44[:, :rmvpe.resampled_length(y48.shape[-1], 48000, 44100)]
    for keyshift in (0, -3.2):
        got = voc.extract(y48.to(DEV), 48000, keyshift=keyshift)
        ref = mel64(y44, 512, keyshift).transpose(1, 2)
        assert got.shape == ref.shape
        d = got.cpu().double() - ref
        report.record("vocoder/extract48k_ks%g" % keyshift, max=d.abs().max().item(), rms=d.pow(2).mean().sqrt().item())
        assert d.abs().max().item() < 5 * TOL_MAX and d.pow(2).mean().sqrt().item() < 5 * TOL_RMS
    y44d = y44.float().to(DEV).requires_grad_()
    m = voc.extract(y44d, 44100)                                # keyshift 0 keeps get_mel's CUDA backward
    m.sum().backward()
    assert y44d.grad is not None and torch.isfinite(y44d.grad).all()
    with pytest.raises(NotImplementedError, match="resampling"):
        voc.extract(y48.to(DEV).requires_grad_(), 48000)


@pytest.mark.parametrize("name", [n for n in mk.CASES if mk.CASES[n]["model"] == "small" and
                                  not mk.CASES[n].get("weight_norm")])
def test_vocoder_infer_replays_the_generator_goldens(tmp_path, name):
    d = np.load(mk.path(name))
    rand_ini, noise = mk.draws(d)
    mel = torch.from_numpy(d["x"]).transpose(1, 2).to(DEV)        # [B, nF, 128]
    f0 = torch.from_numpy(d["f0"])[..., None].to(DEV)
    f0 = torch.cat([f0, f0[:, -1:]], 1)                            # longer f0 is cut to the mel's frames
    ckpt = _write_vocoder(tmp_path, {})
    voc = pkg.Vocoder("nsf-hifigan", ckpt, device=DEV)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        voc.infer(mel[:, :1], f0)                                  # builds the generator from config.json and ckpt
    model = voc.model
    # substitute the reference's draws, as tests/test_gpu_hifigan.py's replay does
    model.forward = functools.partial(type(model).forward, model, rand_ini=rand_ini.to(DEV), noise=noise.to(DEV))
    out = voc.infer(mel, f0).cpu().double()
    ref = torch.from_numpy(d["out64"])
    rel = (out - ref).pow(2).mean().sqrt().item() / ref.pow(2).mean().sqrt().item()
    report.record("vocoder/infer/" + name, rel_rms=rel)
    assert out.shape == ref.shape and rel < 1.5e-5, rel                # tests/test_gpu_hifigan.py's GEN_RMS
    # 'nsf-hifigan-log10' scales by 0.434294 before vocoding: the plain vocoder's bits for 0.434294 * mel
    log10 = pkg.Vocoder("nsf-hifigan-log10", ckpt, device=DEV)
    log10.model = model
    assert torch.equal(log10.infer(mel, f0), voc.infer(0.434294 * mel, f0))
