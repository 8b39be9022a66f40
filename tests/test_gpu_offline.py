"""OfflineVC / OfflineReflowVC (ddsp_svc_b200/offline.py) on the GPU: the Slicer's RMS kernel against float64 and the
goldens' chunks, and whole-file conversions against main.py's / main_reflow.py's own loops over the same modules
(tests/offline_oracle.py) with the same torch seed -- every segment's output bit for bit, the assembled waveform within
one fp32 ulp of the float64 result and only on faded samples.  Synthetic seeded checkpoints (bench_realtime and
bench_realtime_reflow's writers)."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch
import yaml

from bench_realtime import write_synthetic
from bench_realtime_reflow import write_synthetic_reflow
from ddsp_svc_b200 import frontend, offline
from ddsp_svc_b200.offline import OfflineReflowVC, OfflineVC
from tests import offline_oracle as oo
from tests import report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "offline_slicer.npz"))
# 20-40 s clips with 2-4 pauses (a short gap, one up to twice max_sil_kept, one below min_interval, a trailing one)
CLIPS = {"three_pauses": [("v", 6.0), ("s", 1.0), ("v", 6.0), ("s", 7.0), ("v", 5.5), ("s", 0.2), ("v", 4.0)],
         "two_pauses": [("s", 0.5), ("v", 8.0), ("s", 2.5), ("v", 7.0), ("s", 3.0)],
         "four_pauses": [("v", 5.5), ("s", 0.6), ("v", 5.5), ("s", 1.2), ("v", 6.0), ("s", 0.4), ("v", 5.2),
                         ("s", 0.8), ("v", 5.0)]}


def quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


@pytest.fixture(scope="module")
def ddsp_ckpt(tmp_path_factory):
    return quiet(write_synthetic, str(tmp_path_factory.mktemp("offline_ddsp")), "CombSubSuperFast")


@pytest.fixture(scope="module")
def reflow_ckpt(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("offline_reflow"))
    model_path, rmvpe_path = quiet(write_synthetic_reflow, d, n_chans=128, n_layers=2, encoder="hubertsoft")
    cfg_path = os.path.join(d, "config.yaml")
    with open(cfg_path) as f:
        cfg = yaml.safe_load(f)
    cfg["model"]["t_start"] = 0.3                                   # main_reflow.py's floor for a given t_start
    cfg["infer"] = {"method": "rk4", "infer_step": 2}               # what 'auto' reads
    with open(cfg_path, "w") as f:
        yaml.safe_dump(cfg, f)
    return model_path, rmvpe_path


@pytest.fixture(scope="module")
def vc_enh(ddsp_ckpt):
    return quiet(OfflineVC, ddsp_ckpt[0], device=DEV, rmvpe_ckpt=ddsp_ckpt[1])


@pytest.fixture(scope="module")
def vc_raw(ddsp_ckpt):
    return quiet(OfflineVC, ddsp_ckpt[0], device=DEV, enhance=False, rmvpe_ckpt=ddsp_ckpt[1])


@pytest.fixture(scope="module")
def rf(reflow_ckpt):
    rf = quiet(OfflineReflowVC, reflow_ckpt[0], device=DEV, rmvpe_ckpt=reflow_ckpt[1])
    # one call first: the first Unit2Wav call after loading has been seen to differ from later seeded calls (DESIGN §8)
    x = torch.from_numpy(oo.speech([("v", 3.0)], 44100, seed=0)).to(DEV)
    quiet(rf.render, x, 44100, infer_step=1, method="euler", t_start=0.5, segments=[(0, 200)])
    return rf


def clip(name, sr=44100):
    return oo.speech(CLIPS[name], sr, seed=sorted(CLIPS).index(name) + 11)


def test_slicer_rms_at_60_s_against_float64():
    sr = 44100
    p = offline.SlicerParams(sr)
    y = oo.speech([("v", 20.0), ("s", 4.0), ("v", 20.0), ("s", 1.0), ("v", 15.0)], sr, seed=5)
    assert y.shape[0] == 60 * sr
    got = frontend.slicer_rms(torch.from_numpy(y).to(DEV), p.win, p.hop).cpu().numpy()
    y64 = np.pad(y.astype(np.float64), p.win // 2)
    n = 1 + y.shape[0] // p.hop
    want = np.sqrt(np.mean(y64[np.arange(p.win)[None] + p.hop * np.arange(n)[:, None]] ** 2, 1))
    assert got.shape == (n,)
    rel = float(np.max(np.abs(got - want) / want))
    report.record("offline/slicer_rms_60s", max_rel=rel)
    assert rel < 1e-6
    again = frontend.slicer_rms(torch.from_numpy(y).to(DEV), p.win, p.hop).cpu().numpy()
    assert np.array_equal(got, again)                                # no atomics: bit-identical run to run


@pytest.mark.parametrize("name,sr", [(n, sr) for sr in oo.SLICER_RATES for n in sorted(oo.SLICER_CASES)])
def test_device_rms_reproduces_the_golden_chunks(name, sr):
    audio = oo.slicer_case(name, sr)
    p = offline.SlicerParams(sr)
    rms = frontend.slicer_rms(torch.from_numpy(audio).to(DEV), p.win, p.hop).cpu().numpy()
    tags = [] if audio.shape[0] <= p.min_length else offline.silence_tags(rms, p)
    chunks = offline.slicer_chunks(tags, audio.shape[0], p.hop)
    assert np.array_equal(np.array([[b, e, int(s)] for b, e, s in chunks], dtype=np.int64),
                          GOLD["%s_%d_chunks" % (name, sr)])
    split = offline.split_frames(chunks, oo.SPLIT_HOP[sr])
    assert np.array_equal(np.array(split, dtype=np.int64).reshape(-1, 2), GOLD["%s_%d_split" % (name, sr)])


def fade_mask(vc, rendered, out_sr, total):
    plan, n = offline.assembly_plan([s for s, _ in rendered], [o.numel() for _, o in rendered], vc.block_size, out_sr,
                                    vc.model_sr)
    assert n == total
    m = np.zeros(total, bool)
    for idx, fade in plan:
        m[idx:idx + fade] = True
    return m


def check_against_loop(tag, vc, rendered, out, want, want_outs, out_sr):
    assert len(rendered) == len(want_outs) >= 2
    for (_, got), ref in zip(rendered, want_outs):
        assert torch.equal(got.cpu(), torch.from_numpy(ref))         # same calls, same draws: a difference is a bug
    got = out.cpu().numpy()
    assert got.shape == want.shape
    ref32 = want.astype(np.float32)
    ulp = np.abs(got.view(np.int32).astype(np.int64) - ref32.view(np.int32).astype(np.int64))
    fades = fade_mask(vc, rendered, out_sr, got.shape[0])
    report.record("offline/" + tag, fade_samples=int(fades.sum()), max_ulp=int(ulp.max()))
    assert fades.any()
    assert ulp.max() <= 1 and not (ulp[~fades] > 0).any()


@pytest.mark.parametrize("enhance,key,eak,mix", [(True, 0, 0, None), (True, 3, "auto", None), (False, -2, 0, None),
                                                 (True, 1, 2, {1: 0.25, 2: 0.75})])
def test_convert_matches_main_py(vc_enh, vc_raw, enhance, key, eak, mix):
    vc = vc_enh if enhance else vc_raw
    name = "three_pauses" if enhance else "four_pauses"
    audio = clip(name)
    x = torch.from_numpy(audio).to(DEV)
    segments = vc.split(x, 44100)
    kw = dict(key=key, spk_id=2, spk_mix_dict=mix, threhold=-50)
    torch.manual_seed(3)
    rendered, out_sr = quiet(vc.render, x, 44100, enhancer_adaptive_key=eak, segments=segments, **kw)
    out = vc.assemble(rendered, out_sr)
    torch.manual_seed(3)
    want, want_sr, want_outs = quiet(oo.main_loop, vc, audio, 44100, segments, enhancer_adaptive_key=eak, **kw)
    assert out_sr == want_sr == (44100 if not enhance else vc.enhancer.enhancer_sample_rate)
    check_against_loop("main_%s_%s_%s_%s" % (enhance, key, eak, mix is not None), vc, rendered, out, want, want_outs,
                       out_sr)


@pytest.mark.parametrize("infer_step,method,t_start,resolved", [(2, "euler", 0.5, (2, "euler", 0.5)),
                                                                 (3, "rk4", 0.7, (3, "rk4", 0.7)),
                                                                 ("auto", "auto", "auto", (2, "rk4", 0.3)),
                                                                 (3, "euler", 0.1, (3, "euler", 0.3))])
def test_reflow_convert_matches_main_reflow_py(rf, infer_step, method, t_start, resolved):
    assert offline.reflow_settings(rf.args, infer_step, method, t_start) == resolved
    audio = clip("two_pauses")
    x = torch.from_numpy(audio).to(DEV)
    segments = rf.split(x, 44100)
    kw = dict(key=2, spk_id=1, formant_shift_key=1.5)
    torch.manual_seed(4)
    rendered, out_sr = quiet(rf.render, x, 44100, infer_step=infer_step, method=method, t_start=t_start,
                             segments=segments, **kw)
    out = rf.assemble(rendered, out_sr)
    torch.manual_seed(4)
    s, m, t = resolved
    want, want_outs = quiet(oo.main_reflow_loop, rf, audio, 44100, segments, infer_step=s, method=m, t_start=t, **kw)
    assert out_sr == rf.model_sr
    check_against_loop("reflow_%s_%s_%s" % resolved, rf, rendered, out, want, want_outs, out_sr)


def test_given_segments_queue_without_a_sync_and_repeat_bit_for_bit(vc_enh, rf):
    x = torch.from_numpy(clip("two_pauses")).to(DEV)
    for vc, kw in ((vc_enh, dict(enhancer_adaptive_key=1)), (rf, dict(infer_step=2, method="euler", t_start=0.5))):
        segments = vc.split(x, 44100)
        quiet(vc.convert, x, 44100, segments=segments, **kw)                 # warm: tables, packed weights, step rows
        torch.cuda.synchronize()
        outs = []
        for _ in range(2):
            torch.manual_seed(9)
            torch.cuda.set_sync_debug_mode("error")
            try:
                out, _ = vc.convert(x, 44100, segments=segments, **kw)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            outs.append(out.cpu())
        assert torch.equal(outs[0], outs[1])
        torch.manual_seed(9)
        rendered, out_sr = vc.render(x, 44100, segments=segments, **kw)
        assert torch.equal(vc.assemble(rendered, out_sr).cpu(), outs[0])      # convert = render + assemble


def test_convert_splits_by_itself(vc_raw):
    x = torch.from_numpy(clip("four_pauses")).to(DEV)
    segments = vc_raw.split(x, 44100)
    assert len(segments) >= 3
    torch.manual_seed(1)
    a, _ = vc_raw.convert(x, 44100)
    torch.manual_seed(1)
    b, _ = vc_raw.convert(x, 44100, segments=segments)
    assert torch.equal(a, b)


def test_value_errors(vc_raw, ddsp_ckpt, rf):
    x48 = torch.from_numpy(oo.speech([("v", 6.0)], 48000, seed=1)).to(DEV)
    with pytest.raises(ValueError, match="integer hop"):
        vc_raw.convert(x48, 48000)                       # 512 * 48000 / 44100 is not an integer
    with pytest.raises(ValueError, match="integer hop"):
        vc_raw.split(x48, 48000)
    with pytest.raises(ValueError, match="CUDA device"):
        OfflineVC(ddsp_ckpt[0], device="cpu", rmvpe_ckpt=ddsp_ckpt[1])
    with pytest.raises(ValueError, match="rmvpe"):
        OfflineVC(ddsp_ckpt[0], device=DEV, rmvpe_ckpt=ddsp_ckpt[1], pitch_extractor="crepe")
    x = torch.from_numpy(clip("two_pauses")).to(DEV)
    with pytest.raises(ValueError, match="negative"):
        rf.convert(x, 44100, infer_step=-1, method="euler")
    with pytest.raises(ValueError, match="mono"):
        vc_raw.convert(x.cpu(), 44100)
    with pytest.raises(ValueError, match="frame range"):
        vc_raw.convert(x, 44100, segments=[(0, 10 ** 6)])
    with pytest.raises(ValueError, match="cross-fade"):
        vc_raw.assemble([(0, torch.zeros(600, device=DEV)), (1, torch.zeros(3, device=DEV))], 44100)
