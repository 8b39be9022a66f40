"""BatchedRealtimeVC (ddsp_svc_b200/realtime.py) on the GPU: every row against a single RealtimeVC with that session's
settings, input and draws over consecutive blocks; rows independent of each other bit for bit; graph replay against
the eager batched session; replays without hidden synchronisation; update() and reset() without recapture; the batched
kernels against the single-session ones row by row.  Synthetic seeded checkpoints
(conversion_fixtures.write_synthetic)."""
import functools
import types

import numpy as np
import pytest
import torch

from conversion_fixtures import build_session, copy_draws, quiet, write_synthetic
from ddsp_svc_b200 import frontend, ops
from ddsp_svc_b200 import realtime as rt
from ddsp_svc_b200.realtime import BatchedRealtimeVC, RealtimeVC
from tests import report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_BLOCKS = 5
SESSIONS = [dict(spk_id=1, pitch_adjust=0.0, threhold=-45),
            dict(spk_id=2, pitch_adjust=5.0, threhold=-30),
            dict(spk_id=1, pitch_adjust=-4.0, threhold=-60, use_spk_mix=True, spk_mix_dict={1: 0.3, 2: 0.7})]


@pytest.fixture(scope="module", params=["Sins", "CombSubSuperFast"])
def ckpt(request, tmp_path_factory):
    return quiet(write_synthetic, str(tmp_path_factory.mktemp(request.param)), request.param)


batched = functools.partial(build_session, BatchedRealtimeVC, sessions=SESSIONS)


def single(ckpt, settings, **kw):
    return build_session(RealtimeVC, ckpt, **settings, **kw)


def voice(n, sr, f, seed):
    """a clearly periodic voice (vibrato around f Hz) plus a little noise: its SOLA correlation peak is sharp"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = 0.3 * np.sin(2 * np.pi * (f * t + 0.2 * f / 9 * np.sin(2 * np.pi * 5 * t))) + 0.01 * rng.standard_normal(n)
    return x.astype(np.float32)


def inputs(s, seed=0, n_blocks=N_BLOCKS):
    """[n_blocks] of [N, block, 2]: row i a voice at its own pitch"""
    x = np.stack([voice(n_blocks * s.block, s.sr, 150 + 40 * i, seed + i) for i in range(s.n)])
    x = np.stack([x, 0.5 * x], 2)
    return [x[:, k * s.block:(k + 1) * s.block] for k in range(n_blocks)]


def record_shifts(monkeypatch):
    """the shifts the eager single sessions compute, in call order"""
    shifts, sola = [], ops.rt_sola

    def rec(x, buf, search):
        s = sola(x, buf, search)
        shifts.append(int(s.item()))
        return s
    monkeypatch.setattr(rt.ops, "rt_sola", rec)
    return shifts


def rel_rms(got, want):
    rms = np.sqrt(np.mean(want.astype(np.float64) ** 2))
    return rms, np.sqrt(np.mean((got.astype(np.float64) - want) ** 2)) / max(rms, 1e-30)


@pytest.mark.parametrize("pv,key", [(False, 0), (True, 0), (False, 3), (True, 3)])
def test_rows_match_single_sessions(ckpt, monkeypatch, pv, key):
    b = batched(ckpt, graph=False, use_phase_vocoder=pv, enhancer_adaptive_key=key)
    ones = [single(ckpt, c, graph=False, use_phase_vocoder=pv, enhancer_adaptive_key=key) for c in SESSIONS]
    for i, one in enumerate(ones):
        copy_draws(one, b, row=i)                                    # one takes row i of b's draws
    shifts = record_shifts(monkeypatch)
    for k, x in enumerate(inputs(b)):
        got = b.process(x)
        assert got.shape == (b.n, b.block, 2) and got.dtype == np.float32
        b_shift = b.shift.cpu().numpy()
        del shifts[:]
        for i, one in enumerate(ones):
            want = one.process(x[i])
            rms, rel = rel_rms(got[i], want)
            report.record("realtime/batch/%s_%s_%d_%d" % (pv, key, k, i), rel_rms=rel)
            assert rms > 0 and rel < 1e-5, (k, i, rel)
        assert shifts == list(b_shift), (k, shifts, b_shift)


def test_rows_are_independent(ckpt):
    """changing, zeroing or reset()-ing row 1 leaves rows 0 and 2 bit-identical (fixed draws in every run)"""
    runs, draws = [], None
    for variant in ("base", "changed", "zeroed", "reset"):
        b = batched(ckpt, graph=True)
        if draws is None:
            g = torch.Generator(device=DEV).manual_seed(0)
            draws = types.SimpleNamespace(**{name: torch.randn(getattr(b, name).shape, device=DEV, generator=g)
                                             for name in ("noise", "gen_rand_ini", "gen_noise")})
        copy_draws(b, draws)
        outs = []
        for k, x in enumerate(inputs(b)):
            x = x.copy()
            if variant == "changed":
                x[1] = np.random.default_rng(k).standard_normal(x[1].shape).astype(np.float32)
            elif variant == "zeroed":
                x[1] = 0
            elif variant == "reset" and k == 2:
                b.reset(1)
            outs.append(b.process(x))
        runs.append(np.stack(outs))
    for r in runs[1:]:
        assert r[:, [0, 2]].tobytes() == runs[0][:, [0, 2]].tobytes()
    assert not np.array_equal(runs[1][:, 1], runs[0][:, 1])


@pytest.mark.parametrize("pv", [False, True])
def test_graph_replay_is_bit_identical_to_eager(ckpt, pv):
    g = batched(ckpt, graph=True, use_phase_vocoder=pv, enhancer_adaptive_key=3)
    e = batched(ckpt, graph=False, use_phase_vocoder=pv, enhancer_adaptive_key=3)
    copy_draws(e, g)
    for x in inputs(g, seed=1):
        assert np.array_equal(g.process(x), e.process(x))


def test_replays_do_not_synchronise(ckpt):
    s = batched(ckpt, graph=True, enhancer_adaptive_key=2)
    xs = inputs(s, seed=2)
    s.process(xs[0])                                                 # captures A and B
    torch.cuda.synchronize()
    for x in xs[1:3]:
        torch.cuda.set_sync_debug_mode("error")
        try:
            s.upload(x)
            s.run_a()
            s.run_b()
            s.update(1, pitch_adjust=2.0, threhold=-50)
            s.reset(0)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        s.stream.synchronize()                                       # the blocks' output copy


def test_update_matches_fresh_session(ckpt):
    """after update(i, ...) the next block equals a session built with the new settings and the same history, and the
    graphs are the ones captured before"""
    new = [dict(SESSIONS[0]), dict(spk_id=1, pitch_adjust=-3.0, threhold=-40, use_spk_mix=True,
                                  spk_mix_dict={1: 0.5, 2: 0.5}), dict(SESSIONS[2])]
    a = batched(ckpt, graph=True)
    f = batched(ckpt, sessions=new, graph=True)
    copy_draws(f, a)
    xs = inputs(a, seed=3)
    a.process(xs[0])
    graphs = (a.graph_a, a.graph_b)
    for x in xs[1:3]:                                                # the same ring and SOLA history in f
        a.process(x)
    f.ring.copy_(a.ring)
    f.sola_buffer.copy_(a.sola_buffer)
    a.update(1, **{k: new[1][k] for k in ("spk_id", "pitch_adjust", "threhold", "use_spk_mix", "spk_mix_dict")})
    for x in xs[3:]:
        assert np.array_equal(a.process(x), f.process(x))
    assert (a.graph_a, a.graph_b) == graphs


def test_reset_matches_fresh_single_session(ckpt):
    b = batched(ckpt, graph=True)
    xs = inputs(b, seed=4, n_blocks=6)
    for x in xs[:2]:
        b.process(x)
    b.reset(2)
    one = single(ckpt, SESSIONS[2], graph=False)
    copy_draws(one, b, row=2)
    for x in xs[2:]:
        got = b.process(x)
        rms, rel = rel_rms(got[2], one.process(x[2]))
        assert rms > 0 and rel < 1e-5, rel


def test_batched_kernels_equal_single_kernels_per_row():
    """rt_f0_regrid_batch, rt_sola_batch, rt_crossfade_batch and volume_mask_rows against the single-session ops on
    each row, bit for bit"""
    torch.manual_seed(0)
    N, n10, n_frames, cf, search, block = 5, 241, 200, 1764, 441, 13230
    f0 = (220 * 2 ** (0.3 * torch.randn(N, n10, device=DEV))).float()
    f0[torch.rand(N, n10, device=DEV) < 0.3] = 0
    f0[1] = 0
    post = torch.tensor([1.0, 2 ** (5 / 12), 0.5, 2 ** (-7 / 12), 1.25], dtype=torch.float32, device=DEV)
    got = ops.rt_f0_regrid_batch(f0, 0.01, n_frames, 512 / 44100, rmvpe=True, pad=9, f0_min=50.0, post_scale=post)
    for i in range(N):
        want = ops.rt_f0_regrid(f0[i].contiguous(), 0.01, n_frames, 512 / 44100, rmvpe=True, pad=9, f0_min=50.0,
                                post_scale=float(post[i]))
        assert torch.equal(got[i], want)
    audio = torch.randn(N, 3 * block, device=DEV)
    temp = audio[:, 100:100 + block + cf + search]
    buf = torch.stack([temp[i, s:s + cf] for i, s in enumerate([0, search, 17, 300, search])]).contiguous()
    shift = ops.rt_sola_batch(temp, buf, search)
    assert shift.tolist() == [0, search, 17, 300, search]
    fi = torch.sin(np.pi * torch.arange(0, 1, 1 / cf, device=DEV) / 2) ** 2
    for pv in (False, True):
        out, nxt = ops.rt_crossfade_batch(temp, shift, search, buf, fi, 1 - fi, block, pv)
        for i in range(N):
            x = temp[i].contiguous()
            s1 = ops.rt_sola(x, buf[i].contiguous(), search)
            assert int(s1) == int(shift[i])
            o1, n1 = ops.rt_crossfade(x, s1, search, buf[i].contiguous(), fi, 1 - fi, block, pv)
            assert torch.equal(out[i], o1) and torch.equal(nxt[i], n1)
    vol = frontend.volume_extract(audio * torch.linspace(0, 1, 3 * block, device=DEV), 512)
    dbs = [-45, -30, -60, -20, -45]
    thr = torch.tensor([frontend.mask_threshold(d) for d in dbs], dtype=torch.float32, device=DEV)
    m = frontend.volume_mask_rows(vol, thr)
    for i in range(N):
        assert torch.equal(m[i], frontend.volume_mask(vol[i:i + 1], dbs[i])[0])


def test_errors(ckpt):
    with pytest.raises(ValueError, match="own"):
        batched(ckpt, enhancer_adaptive_key="auto")
    with pytest.raises(ValueError, match="at least one"):
        batched(ckpt, sessions=[])
    with pytest.raises(ValueError, match="CUDA"):
        BatchedRealtimeVC(ckpt[0], SESSIONS, rmvpe_ckpt=ckpt[1], device="cpu")
    s = batched(ckpt, graph=False)
    with pytest.raises(ValueError, match="indata"):
        s.process(np.zeros((2, s.block, 2), np.float32))
    with pytest.raises(ValueError, match="indata"):
        s.process(np.zeros((3, s.block - 1), np.float32))
    with pytest.raises(IndexError):
        s.update(3, pitch_adjust=1.0)
    with pytest.raises(ValueError, match="unknown"):
        s.update(0, key=1.0)
