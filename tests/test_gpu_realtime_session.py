"""RealtimeVC (ddsp_svc_b200/realtime.py) on the GPU: the eager session against gui.py's order on the same modules and
noise over consecutive blocks (the SOLA state carries over), graph replay against the eager session bit for bit, and
replays without hidden synchronisation.  Synthetic seeded checkpoints (bench_realtime.write_synthetic)."""
import contextlib
import io

import numpy as np
import pytest
import torch

from bench_realtime import GuiBlock, write_synthetic
from ddsp_svc_b200.realtime import RealtimeVC
from tests import report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_BLOCKS = 5


@pytest.fixture(scope="module", params=["Sins", "CombSubSuperFast"])
def ckpt(request, tmp_path_factory):
    d = tmp_path_factory.mktemp(request.param)
    with contextlib.redirect_stdout(io.StringIO()):
        return write_synthetic(str(d), request.param)


def session(ckpt, **kw):
    model_path, rmvpe_path = ckpt
    with contextlib.redirect_stdout(io.StringIO()):
        return RealtimeVC(model_path, rmvpe_ckpt=rmvpe_path, device=DEV, **kw)


def blocks(s, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(N_BLOCKS * s.block) / s.sr
    x = 0.3 * np.sin(2 * np.pi * (180 * t + 20 * np.sin(2 * np.pi * t))) + 0.01 * rng.standard_normal(t.size)
    x = np.stack([x, 0.5 * x], 1).astype(np.float32)
    return [x[i * s.block:(i + 1) * s.block] for i in range(N_BLOCKS)]


@pytest.mark.parametrize("pv,key", [(True, 0), (False, 3), (True, "auto"), (False, "auto")])
def test_eager_session_matches_gui_order(ckpt, pv, key):
    s = session(ckpt, graph=False, use_phase_vocoder=pv, enhancer_adaptive_key=key)
    ref = GuiBlock(s)
    for i, x in enumerate(blocks(s)):
        got = s.process(x)
        with contextlib.redirect_stdout(io.StringIO()), torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            want = ref(x)                                            # reads the noise the session just drew
        assert got.shape == want.shape == (s.block, 2)
        rms = np.sqrt(np.mean(want ** 2))
        rel = np.sqrt(np.mean((got - want) ** 2)) / max(rms, 1e-30)
        report.record("realtime/session/%s_%s_%d" % (pv, key, i), rel_rms=rel)
        assert rms > 0 and rel < 1e-5, (i, rel)


@pytest.mark.parametrize("pv,key", [(True, 0), (False, "auto")])
def test_graph_replay_is_bit_identical_to_eager(ckpt, pv, key):
    g = session(ckpt, graph=True, use_phase_vocoder=pv, enhancer_adaptive_key=key)
    e = session(ckpt, graph=False, use_phase_vocoder=pv, enhancer_adaptive_key=key)
    # the eager session takes the graph session's draws of each block
    e._draw_noise = lambda: e.noise.copy_(g.noise)
    e._draw_enhancer_noise = lambda: (e.gen_rand_ini.copy_(g.gen_rand_ini), e.gen_noise.copy_(g.gen_noise))
    for x in blocks(g, seed=1):
        a = g.process(x)
        b = e.process(x)
        assert np.array_equal(a, b)


def test_replays_do_not_synchronise(ckpt):
    s = session(ckpt, graph=True, enhancer_adaptive_key=2)
    xs = blocks(s, seed=2)
    s.process(xs[0])                                                 # captures A and B[2]
    torch.cuda.synchronize()
    for x in xs[1:3]:
        torch.cuda.set_sync_debug_mode("error")
        try:
            s.upload(x)
            s.run_a()
            s.run_b(s.pick_key())
        finally:
            torch.cuda.set_sync_debug_mode(0)
        s.stream.synchronize()                                       # the block's output copy


def test_other_pitch_extractors_raise(ckpt):
    with pytest.raises(ValueError, match="rmvpe"):
        RealtimeVC(ckpt[0], pitch_extractor_type="crepe", device=DEV)
