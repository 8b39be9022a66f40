"""The reflow cascade Unit2Wav (ddsp_svc_b200/reflow_vocoder.py) on the kernels against the live reference's outputs
(tests/golden/unit2wav_*.npz, tests/golden/make_golden_unit2wav.py), fed the reference's draws; and load_model_vocoder.

Error is relative to the reference run in float64 (``out64``): rms(got - out64) / rms(out64), bounded by
max(1e-5, 3 x the reference's own fp32 error against out64).  Measured errors go through tests/report.py
(B2D_PARITY_REPORT)."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch
import yaml

import ddsp_svc_b200 as pkg
from tests import report
from tests.golden import make_golden_unit2wav as mk

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def rel_rms(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.sqrt(np.mean((a - b) ** 2)) / np.sqrt(np.mean(b ** 2)))


@pytest.fixture(scope="module")
def vocoder(tmp_path_factory):
    ckpt = mk.write_vocoder(str(tmp_path_factory.mktemp("voc")))
    return pkg.Vocoder("nsf-hifigan", ckpt, device=DEV)


@pytest.mark.parametrize("name", list(mk.CASES))
def test_matches_the_reference(name, vocoder):
    c = mk.CASES[name]
    d = dict(np.load(mk.path(name)))
    m = mk.MODELS[c["model"]]
    net = pkg.Unit2Wav(44100, 512, 2048, mk.N_UNIT, mk.N_SPK, True, 128, m["n_layers"], m["n_chans"])
    net.load_state_dict(mk.state_dict(c["model"]), strict=True)
    net = net.to(DEV).eval()
    dr = {k: v.to(DEV) for k, v in mk.draws(d, name).items()}
    g = lambda k: torch.from_numpy(d[k]).to(DEV)
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        got = net(g("units"), g("f0"), g("volume"), spk_id=g("spk_id"), aug_shift=g("aug_shift"), vocoder=vocoder,
                  infer=True, return_wav=c["return_wav"], infer_step=c["steps"], method=c["method"],
                  t_start=c["t_start"], silence_front=c["silence_front"], use_tqdm=False,
                  ddsp_noise=dr["ddsp_noise"], reflow_noise=dr.get("reflow_noise"), rand_ini=dr.get("rand_ini"),
                  sine_noise=dr.get("sine_noise"))
    assert tuple(got.shape) == d["out32"].shape
    err, ref_err = rel_rms(got.cpu().numpy(), d["out64"]), rel_rms(d["out32"], d["out64"])
    bound = max(1e-5, 3 * ref_err)
    report.record("unit2wav/%s" % name, rel_rms=err, reference_fp32_rel_rms=ref_err, bound=bound)
    assert err < bound, (err, ref_err)


def write_checkpoint(d, model_type):
    ckpt = mk.write_vocoder(d)
    cfg = {"data": {"sampling_rate": 44100, "block_size": 512, "encoder_out_channels": mk.N_UNIT},
           "model": {"type": model_type, "win_length": 2048, "n_layers": 2, "n_chans": 128, "use_pitch_aug": True,
                     "n_spk": mk.N_SPK},
           "vocoder": {"type": "nsf-hifigan", "ckpt": ckpt}}
    with open(os.path.join(d, "config.yaml"), "w") as f:
        yaml.safe_dump(cfg, f)
    path = os.path.join(d, "model.pt")
    torch.save({"model": mk.state_dict("w128")}, path)
    return path


def test_load_model_vocoder(tmp_path):
    path = write_checkpoint(str(tmp_path), "RectifiedFlow")
    with contextlib.redirect_stdout(io.StringIO()):
        model, vocoder, args = pkg.load_model_vocoder(path, device=DEV)
    assert isinstance(model, pkg.Unit2Wav) and not model.training and args.model.type == "RectifiedFlow"
    assert vocoder.dimension == 128 and vocoder.vocoder_hop_size == 512
    want = mk.state_dict("w128")
    for k, v in model.state_dict().items():
        assert v.device.type == "cuda" and torch.equal(v.cpu(), want[k]), k


def test_load_model_vocoder_rejects_other_types(tmp_path):
    path = write_checkpoint(str(tmp_path), "DiffusionNew")
    with pytest.raises(ValueError, match="Unknown Model"):
        pkg.load_model_vocoder(path, device=DEV)
