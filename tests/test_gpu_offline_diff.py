"""OfflineDiffVC (ddsp_svc_b200/offline.py) on the GPU against main_diff.py's loop and batch_infer.py's infer() restated
over the same modules (tests/offline_diff_oracle.py) with the same torch seed.

Every comparison runs on the FIRST call after construction, with no warm-up: each test builds its converter afresh.
Each segment's output is bit-identical to the loop's, the assembled waveform is within one fp32 ulp of the float64
result and differs only on faded samples, and convert_whole equals infer() bit for bit.  The cases reach every mode of
each model type under both drivers ('ddsp': the external DDSP model's mel; 'input_mel'; 'none'), DDPM and four samplers
at speedup 10 or more, k_step above k_step_max, formant keys 0 and +-3, a speaker mix and an explicit diffusion speaker.
Checkpoints are synthetic and seeded (conversion_fixtures.write_synthetic_diff, small widths), with a CombSubSuperFast
DDSP checkpoint that fits and a CombSub one at block_size 256 that does not."""
import os

import numpy as np
import pytest
import torch
import yaml

from conversion_fixtures import DDSP_MODELS, quiet, write_synthetic_diff, write_synthetic_reflow
from ddsp_svc_b200 import dropin, offline
from ddsp_svc_b200.offline import OfflineDiffVC
from tests import offline_diff_oracle as odo
from tests import offline_oracle as oo
from tests import report
from tests.test_gpu_offline import check_against_loop, clip

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TYPES = ("Diffusion", "DiffusionNew", "DiffusionFast")
MIX = {1: 0.25, 2: 0.75}


@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    """{model type: (diffusion path, rmvpe path)}, the fitting DDSP checkpoint and the one at block_size 256"""
    out = {}
    for kind in TYPES:
        d = str(tmp_path_factory.mktemp("offline_diff_" + kind))
        ddsp, diff, rmvpe = quiet(write_synthetic_diff, d, kind, n_chans=128, n_layers=2, encoder="hubertsoft",
                                  ddsp="CombSubSuperFast")
        cfg_path = os.path.join(d, "diff", "config.yaml")
        with open(cfg_path) as f:
            cfg = yaml.safe_load(f)
        cfg["infer"] = {"speedup": 10, "method": "dpm-solver"}              # what 'auto' reads
        with open(cfg_path, "w") as f:
            yaml.safe_dump(cfg, f)
        out[kind] = diff, rmvpe
    # a CombSub DDSP model at block_size 256 beside the same front
    bad_dir = os.path.join(os.path.dirname(os.path.dirname(ddsp)), "ddsp_block256")
    os.makedirs(bad_dir, exist_ok=True)
    with open(os.path.join(os.path.dirname(ddsp), "config.yaml")) as f:
        dcfg = yaml.safe_load(f)
    dcfg["data"]["block_size"] = 256
    dcfg["model"] = DDSP_MODELS["CombSub"]
    with open(os.path.join(bad_dir, "config.yaml"), "w") as f:
        yaml.safe_dump(dcfg, f)
    bad = os.path.join(bad_dir, "model.pt")
    torch.save({"model": dropin.build_model(dropin.DotDict(dcfg)).state_dict()}, bad)
    return out, ddsp, bad


def make(ckpts, kind, ddsp):
    """a fresh converter: ddsp None, 'fit' or 'block256' (which warns and is dropped)"""
    paths, fit, bad = ckpts
    diff, rmvpe = paths[kind]
    path = {None: None, "fit": fit, "block256": bad}[ddsp]
    if ddsp == "block256":
        with pytest.warns(UserWarning, match="data.block_size differs"):
            vc = quiet(OfflineDiffVC, diff, path, device=DEV, rmvpe_ckpt=rmvpe)
        assert vc.ddsp_model is None and vc.ddsp_args is not None
        return vc
    return quiet(OfflineDiffVC, diff, path, device=DEV, rmvpe_ckpt=rmvpe)


# (model type, DDSP checkpoint, k_step, speedup, method, formant key, mix, diff_spk_id, mode under main_diff.py)
SLICED = [
    ("Diffusion", None, None, 100, "dpm-solver", 0, None, "auto", "none"),
    ("Diffusion", None, 20, 1, "ddim", 3, None, "1", "input_mel"),
    ("Diffusion", "fit", 40, 10, "ddim", -3, MIX, "auto", "ddsp"),
    ("Diffusion", "block256", 40, 100, "pndm", 0, None, "auto", "none"),
    ("DiffusionNew", None, None, "auto", "auto", 0, None, "auto", "none"),
    ("DiffusionNew", "fit", 150, 10, "unipc", 3, MIX, "auto", "ddsp"),
    ("DiffusionNew", "block256", 8, 1, "dpm-solver", 0, None, "1", "none"),
    ("DiffusionFast", None, 40, 10, "ddim", -3, None, "auto", "none"),
    ("DiffusionFast", "fit", 150, 10, "dpm-solver", 0, None, "1", "ddsp"),
    ("DiffusionFast", "block256", 8, 1, "ddim", 3, None, "auto", "none"),
]


@pytest.mark.parametrize("kind,ddsp,k_step,speedup,method,fsk,mix,diff_spk,mode", SLICED,
                         ids=["%s-%s-k%s-%s-%s-f%s" % c[:6] for c in SLICED])
def test_convert_matches_main_diff_py(ckpts, kind, ddsp, k_step, speedup, method, fsk, mix, diff_spk, mode):
    vc = make(ckpts, kind, ddsp)
    s = vc.settings(k_step, speedup, method, diff_spk)
    assert s.mode == mode
    if kind != "Diffusion" and k_step is not None:
        assert s.k_step == min(k_step, 100)
    audio = clip("two_pauses")
    x = torch.from_numpy(audio).to(DEV)
    segments = vc.split(x, 44100)
    kw = dict(key=2, spk_id=2, spk_mix_dict=mix, threhold=-50, formant_shift_key=fsk)
    torch.manual_seed(5)
    rendered, out_sr = quiet(vc.render, x, 44100, diff_spk_id=diff_spk, speedup=speedup, method=method, k_step=k_step,
                             segments=segments, **kw)
    out = vc.assemble(rendered, out_sr)
    torch.manual_seed(5)
    want, want_outs = quiet(odo.main_diff_loop, vc, audio, 44100, segments, s, **kw)
    assert out_sr == vc.model_sr == 44100
    assert all(torch.isfinite(o).all() for _, o in rendered)
    check_against_loop("diff_%s_%s_%s_%s" % (kind, ddsp, mode, method), vc, rendered, out, want, want_outs, out_sr)


# (model type, DDSP checkpoint, k_step, formant key, mode under batch_infer.py)
WHOLE = [
    ("Diffusion", None, None, 0, "none"),
    ("Diffusion", None, 30, 3, "input_mel"),
    ("Diffusion", "block256", 30, 0, "input_mel"),
    ("Diffusion", "fit", 30, -3, "ddsp"),
    ("DiffusionNew", None, 150, 0, "none"),
    ("DiffusionNew", "fit", None, 3, "ddsp"),
    ("DiffusionFast", "fit", None, 0, "none"),
    ("DiffusionFast", "fit", 40, -3, "ddsp"),
]


@pytest.mark.parametrize("kind,ddsp,k_step,fsk,mode", WHOLE, ids=["%s-%s-k%s-f%s" % c[:4] for c in WHOLE])
def test_convert_whole_matches_batch_infer_py(ckpts, kind, ddsp, k_step, fsk, mode):
    vc = make(ckpts, kind, ddsp)
    speedup = 100 if kind == "Diffusion" and mode == "none" else 10
    s = vc.settings(k_step, speedup, "dpm-solver", whole=True)
    assert s.mode == mode
    audio = clip("four_pauses")
    x = torch.from_numpy(audio).to(DEV)
    kw = dict(key=-1, spk_id=1, threhold=-50, formant_shift_key=fsk)
    torch.manual_seed(6)
    out, sr = quiet(vc.convert_whole, x, 44100, speedup=speedup, method="dpm-solver", k_step=k_step, **kw)
    torch.manual_seed(6)
    want = quiet(odo.batch_infer, vc, audio, 44100, s, **kw)
    assert sr == 44100 and out.shape == ((audio.shape[0] // 512 + 1) * 512,)
    got = out.cpu().numpy()
    assert np.isfinite(got).all() and np.array_equal(got, want)


@pytest.mark.parametrize("kind", ["DiffusionNew", "DiffusionFast"])
def test_convert_whole_takes_three_minutes_in_one_call(ckpts, kind):
    vc = make(ckpts, kind, None)
    pieces = [("v", 20.0), ("s", 1.5), ("v", 30.0), ("s", 0.5), ("v", 40.0), ("s", 3.0), ("v", 45.0), ("s", 1.0),
              ("v", 39.0)]
    audio = oo.speech(pieces, 44100, seed=31)
    n_frames = audio.shape[0] // 512 + 1
    assert 15000 < n_frames < 16000
    x = torch.from_numpy(audio).to(DEV)
    kw = dict(key=0, spk_id=1, formant_shift_key=0)
    torch.manual_seed(7)
    out, _ = quiet(vc.convert_whole, x, 44100, speedup=10, method="dpm-solver", k_step=100, **kw)
    torch.manual_seed(7)
    want = quiet(odo.batch_infer, vc, audio, 44100, vc.settings(100, 10, "dpm-solver", whole=True), **kw)
    got = out.cpu().numpy()
    report.record("offline_diff/whole_3min_" + kind, frames=n_frames, peak=float(np.abs(got).max()))
    assert got.shape == (n_frames * 512,) and np.isfinite(got).all() and np.abs(got).max() > 0
    assert np.array_equal(got, want)


@pytest.mark.parametrize("kind,ddsp,k_step,fsk", [("Diffusion", None, 20, 3), ("DiffusionNew", "fit", 40, -3)])
def test_given_segments_queue_without_a_sync_and_repeat_bit_for_bit(ckpts, kind, ddsp, k_step, fsk):
    vc = make(ckpts, kind, ddsp)
    x = torch.from_numpy(clip("two_pauses")).to(DEV)
    segments = vc.split(x, 44100)
    kw = dict(formant_shift_key=fsk, speedup=10, method="dpm-solver", k_step=k_step, spk_mix_dict=MIX)
    for call in (lambda: vc.convert(x, 44100, segments=segments, **kw)[0],
                 lambda: vc.convert_whole(x, 44100, **kw)[0]):
        quiet(call)                                       # warm: packed weights, sampler rows, tables
        torch.cuda.synchronize()
        outs = []
        for _ in range(2):
            torch.manual_seed(9)
            torch.cuda.set_sync_debug_mode("error")
            try:
                out = call()
            finally:
                torch.cuda.set_sync_debug_mode(0)
            outs.append(out.cpu())
        assert torch.equal(outs[0], outs[1])


def test_value_errors(ckpts):
    vc = make(ckpts, "DiffusionNew", None)
    x48 = torch.from_numpy(oo.speech([("v", 6.0)], 48000, seed=1)).to(DEV)
    with pytest.raises(ValueError, match="integer hop"):
        vc.convert(x48, 48000, k_step=20)
    with pytest.raises(ValueError, match="integer hop"):
        vc.convert_whole(x48, 48000, k_step=20)
    paths, fit, _ = ckpts
    diff, rmvpe = paths["DiffusionNew"]
    with pytest.raises(ValueError, match="CUDA device"):
        OfflineDiffVC(diff, fit, device="cpu", rmvpe_ckpt=rmvpe)
    with pytest.raises(ValueError, match="rmvpe"):
        OfflineDiffVC(diff, fit, device=DEV, rmvpe_ckpt=rmvpe, pitch_extractor="harvest")
    x = torch.from_numpy(clip("two_pauses")).to(DEV)
    with pytest.raises(ValueError, match="mono"):
        vc.convert_whole(x.cpu(), 44100)
    with pytest.raises(ValueError, match="frame range"):
        vc.convert(x, 44100, segments=[(0, 10 ** 6)])
    del vc.args["infer"]
    with pytest.raises(ValueError, match="infer.speedup"):
        vc.convert(x, 44100)
    assert offline.diff_settings(vc.args, None, 20, 10, "ddim").k_step == 20


def test_reflow_first_call_matches_main_reflow_py(tmp_path):
    """the first Unit2Wav call after loading equals main_reflow.py's loop under the same seed: the vocoder's generator,
    built on that call, no longer advances torch's CPU generator, from which SineGen's noise seed is drawn"""
    from ddsp_svc_b200.offline import OfflineReflowVC
    model_path, rmvpe_path = quiet(write_synthetic_reflow, str(tmp_path), n_chans=128, n_layers=2, encoder="hubertsoft")
    rf = quiet(OfflineReflowVC, model_path, device=DEV, rmvpe_ckpt=rmvpe_path)
    audio = clip("two_pauses")
    x = torch.from_numpy(audio).to(DEV)
    segments = rf.split(x, 44100)
    kw = dict(key=2, spk_id=1, formant_shift_key=1.5, infer_step=2, method="euler", t_start=0.5)
    torch.manual_seed(4)
    rendered, out_sr = quiet(rf.render, x, 44100, segments=segments, **kw)
    out = rf.assemble(rendered, out_sr)
    torch.manual_seed(4)
    want, want_outs = quiet(oo.main_reflow_loop, rf, audio, 44100, segments, **kw)
    check_against_loop("reflow_first_call", rf, rendered, out, want, want_outs, out_sr)
