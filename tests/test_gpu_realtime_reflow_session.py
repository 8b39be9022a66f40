"""RealtimeReflowVC (ddsp_svc_b200/realtime.py) on the GPU: the eager session against gui_reflow.py's order on the same
modules and draws over consecutive blocks (the SOLA state carries over), graph replay against the eager session bit
for bit, replays without hidden synchronisation, and the session's ValueErrors.  Synthetic seeded checkpoints
(conversion_fixtures.write_synthetic_reflow, a 128 x 2 velocity network and HuBERT-soft units to keep it short)."""
import contextlib
import functools
import io
import os

import numpy as np
import pytest
import torch
import yaml

from conversion_fixtures import GuiReflowBlock, blocks, build_session, copy_draws, quiet, write_synthetic_reflow
from ddsp_svc_b200.realtime import RealtimeReflowVC
from tests import report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ckpt(tmp_path_factory):
    d = tmp_path_factory.mktemp("reflow")
    return quiet(write_synthetic_reflow, str(d), n_chans=128, n_layers=2, encoder="hubertsoft")


session = functools.partial(build_session, RealtimeReflowVC, infer_step=4)
blocks = functools.partial(blocks, quiet_stretch=True)                 # the mask closes in the first block


CASES = {
    "euler_pv": dict(sampling_method="euler", use_phase_vocoder=True),
    "euler_key": dict(sampling_method="euler", formant_shift_key=2.0, pitch_adjust=-3.0),
    "rk4": dict(sampling_method="rk4", infer_step=2, formant_shift_key=-1.5),
    "rk4_pv_t1": dict(sampling_method="rk4", use_phase_vocoder=True, t_start=1.0),
    "euler_t1": dict(sampling_method="euler", t_start=1.0, formant_shift_key=1.0),
    "euler_mix": dict(sampling_method="euler", use_spk_mix=True, spk_mix_dict={1: 0.3, 2: 0.7}),
    "euler_block03": dict(sampling_method="euler", block_time=0.3, extra_time=1.0),
}


@pytest.mark.parametrize("case", list(CASES))
def test_eager_session_matches_gui_reflow_order(ckpt, case):
    s = session(ckpt, graph=False, **CASES[case])
    ref = GuiReflowBlock(s)
    for i, x in enumerate(blocks(s)):
        got = s.process(x)
        with contextlib.redirect_stdout(io.StringIO()), torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            want = ref(x)                                            # reads the draws the session just made
        assert got.shape == want.shape == (s.block, 2)
        rms = np.sqrt(np.mean(want.astype(np.float64) ** 2))
        rel = np.sqrt(np.mean((got.astype(np.float64) - want) ** 2)) / max(rms, 1e-30)
        report.record("realtime_reflow/session/%s_%d" % (case, i), rel_rms=rel)
        assert rms > 0 and rel < 1e-5, (i, rel)


@pytest.mark.parametrize("case", ["euler_pv", "rk4"])
def test_graph_replay_is_bit_identical_to_eager(ckpt, case):
    g = session(ckpt, graph=True, **CASES[case])
    e = session(ckpt, graph=False, **CASES[case])
    copy_draws(e, g)                                                 # the eager session takes g's draws
    for x in blocks(g, seed=1):
        a = g.process(x)
        b = e.process(x)
        assert np.array_equal(a, b)


def test_replays_do_not_synchronise(ckpt):
    s = session(ckpt, graph=True, formant_shift_key=1.0)
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


def test_sampler_issues_no_copy_after_warm_call(ckpt):
    s = session(ckpt, graph=False)
    flow, dev = s.model.reflow_model, torch.device(DEV)
    cond = torch.randn(1, 20, 128, device=dev)
    noise = torch.randn(1, 1, 128, 20, device=dev)
    with torch.no_grad():
        first = flow(cond, gt_spec=cond, infer_step=3, method="rk4", t_start=0.7, noise=noise)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            again = flow(cond, gt_spec=cond, infer_step=3, method="rk4", t_start=0.7, noise=noise)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        other = flow(cond, gt_spec=cond, infer_step=2, method="rk4", t_start=0.7, noise=noise)
        rebuilt = flow(cond, gt_spec=cond, infer_step=3, method="rk4", t_start=0.7, noise=noise)
    assert torch.equal(first, again) and torch.equal(first, rebuilt) and not torch.equal(first, other)


@pytest.mark.parametrize("kw,match", [(dict(pitch_extractor_type="fcpe"), "rmvpe"), (dict(infer_step=0), "infer_step"),
                                      (dict(sampling_method="dpm"), "dpm"), (dict(samplerate=48000), "integer hop")])
def test_invalid_settings_raise(ckpt, kw, match):
    with pytest.raises(ValueError, match=match):
        session(ckpt, **kw)


def test_other_model_types_raise(ckpt, tmp_path):
    model_path, rmvpe_path = ckpt
    with open(os.path.join(os.path.dirname(model_path), "config.yaml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model"]["type"] = "DiffusionNew"
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    torch.save(torch.load(model_path), tmp_path / "model.pt")
    with pytest.raises(ValueError, match="Unknown Model"):
        RealtimeReflowVC(str(tmp_path / "model.pt"), rmvpe_ckpt=rmvpe_path, device=DEV)
