"""RealtimeDiffVC (ddsp_svc_b200/realtime.py) on the GPU: the eager session against gui_diff.py's order on the same
modules and draws over consecutive blocks (the SOLA state carries over), graph replay against the eager session bit
for bit, replays without hidden synchronisation, and the session's ValueErrors.  Synthetic seeded checkpoints
(conversion_fixtures.write_synthetic_diff: 128-channel, 2-layer denoisers and HuBERT-soft units to keep it short)."""
import contextlib
import functools
import gc
import io
import os
import shutil

import numpy as np
import pytest
import torch
import yaml

from conversion_fixtures import GuiDiffBlock, blocks, build_session, copy_draws, quiet, write_synthetic_diff
from ddsp_svc_b200.realtime import RealtimeDiffVC
from tests import report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODELS = {"mel_combsub": ("Diffusion", "CombSub"), "mel_superfast": ("Diffusion", "CombSubSuperFast"),
          "mel_none": ("Diffusion", None), "new": ("DiffusionNew", None), "fast": ("DiffusionFast", None)}


@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    return {name: quiet(write_synthetic_diff, str(tmp_path_factory.mktemp(name)), kind, n_chans=128, n_layers=2,
                        encoder="hubertsoft", ddsp=ddsp) for name, (kind, ddsp) in MODELS.items()}


def session(ckpts, model, **kw):
    return build_session(RealtimeDiffVC, ckpts[model], **dict(dict(k_step=20, diff_acc=5), **kw))


blocks = functools.partial(blocks, quiet_stretch=True)                 # the mask closes in the first block


CASES = {
    "mel_combsub_ddim": ("mel_combsub", dict(diff_method="ddim")),
    "mel_combsub_ddpm": ("mel_combsub", dict(diff_acc=1, k_step=10)),
    "mel_superfast_pndm_pv": ("mel_superfast", dict(diff_method="pndm", use_phase_vocoder=True)),
    "mel_none_dpm": ("mel_none", dict(diff_method="dpm-solver", k_step=400, diff_acc=200)),
    "new_unipc_silence": ("new", dict(diff_method="unipc", diff_silence=True)),
    "new_ddpm_mix": ("new", dict(diff_acc=1, k_step=10, use_spk_mix=True, spk_mix_dict={1: 0.3, 2: 0.7})),
    "new_k0": ("new", dict(k_step=0)),
    "new_ddim_block03": ("new", dict(diff_method="ddim", block_time=0.3, extra_time=1.0)),
    "fast_dpm_pitch": ("fast", dict(diff_method="dpm-solver", pitch_adjust=-3.0)),
    "fast_dpm_silence_pv": ("fast", dict(diff_method="dpm-solver", diff_silence=True, use_phase_vocoder=True)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_eager_session_matches_gui_diff_order(ckpts, case):
    model, kw = CASES[case]
    s = session(ckpts, model, graph=False, **kw)
    ref = GuiDiffBlock(s)
    for i, x in enumerate(blocks(s)):
        got = s.process(x)
        with contextlib.redirect_stdout(io.StringIO()), torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            want = ref(x)                                            # reads the draws the session just made
        assert got.shape == want.shape == (s.block, 2)
        rms = np.sqrt(np.mean(want.astype(np.float64) ** 2))
        rel = np.sqrt(np.mean((got.astype(np.float64) - want) ** 2)) / max(rms, 1e-30)
        report.record("realtime_diff/session/%s_%d" % (case, i), rel_rms=rel)
        assert rms > 0 and rel < 1e-5, (i, rel)


@pytest.mark.parametrize("case", ["mel_superfast_pndm_pv", "fast_dpm_silence_pv", "new_ddpm_mix", "mel_combsub_ddim"])
def test_graph_replay_is_bit_identical_to_eager(ckpts, case):
    model, kw = CASES[case]
    kw = dict(kw, diff_method="ddim") if case == "mel_superfast_pndm_pv" else kw     # DDIM with the phase vocoder
    g = session(ckpts, model, graph=True, **kw)
    e = session(ckpts, model, graph=False, **kw)
    copy_draws(e, g)                                                 # the eager session takes g's draws
    for x in blocks(g, seed=1):
        a = g.process(x)
        b = e.process(x)
        assert np.array_equal(a, b)


def test_capture_runs_without_the_cycle_collector(ckpts):
    """a collection during capture could destroy another session's unreachable graph mid-capture"""
    s = session(ckpts, "new", graph=True)
    seen, stage = [], s._stage

    def watched():
        seen.append(gc.isenabled())
        return stage()
    s._stage = watched
    try:
        s.process(blocks(s)[0])                                      # the warm-up, then the capture
    finally:
        del s._stage
    assert seen == [True, False] and gc.isenabled()


@pytest.mark.parametrize("model", ["mel_combsub", "new"])
def test_replays_do_not_synchronise(ckpts, model):
    s = session(ckpts, model, graph=True, diff_method="dpm-solver")
    xs = blocks(s, seed=2)
    s.process(xs[0])                                                 # captures the block
    torch.cuda.synchronize()
    for x in xs[1:3]:
        torch.cuda.set_sync_debug_mode("error")
        try:
            s.upload(x)
            s.run()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        s.stream.synchronize()                                       # the block's output copy


@pytest.mark.parametrize("model,kw,match", [
    ("new", dict(k_step=200, diff_acc=10), "k_step_max"),
    ("mel_combsub", dict(k_step=0), "k_step"),
    ("new", dict(samplerate=48000), "integer hop"),
    ("new", dict(diff_method="heun"), "diff_method"),
    ("new", dict(k_step=20, diff_acc=11), "diff_acc"),
])
def test_invalid_settings_raise(ckpts, model, kw, match):
    with pytest.raises(ValueError, match=match):
        session(ckpts, model, **kw)


@pytest.mark.parametrize("field,value", [("block_size", 256), ("sampling_rate", 48000), ("encoder", "contentvec768l12")])
def test_mismatched_ddsp_config_raises(ckpts, tmp_path, field, value):
    ddsp_path, diff_path, rmvpe_path = ckpts["mel_combsub"]
    shutil.copy(ddsp_path, tmp_path / "model.pt")
    with open(os.path.join(os.path.dirname(ddsp_path), "config.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["data"][field] = value
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    with pytest.raises(ValueError, match=field):
        RealtimeDiffVC(str(tmp_path / "model.pt"), diff_path, rmvpe_ckpt=rmvpe_path, device=DEV)


def test_other_model_types_raise(ckpts, tmp_path):
    _, diff_path, rmvpe_path = ckpts["new"]
    with open(os.path.join(os.path.dirname(diff_path), "config.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model"]["type"] = "RectifiedFlow"
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    shutil.copy(diff_path, tmp_path / "model.pt")
    with pytest.raises(ValueError, match="Unknown Model"):
        RealtimeDiffVC(None, str(tmp_path / "model.pt"), rmvpe_ckpt=rmvpe_path, device=DEV)
