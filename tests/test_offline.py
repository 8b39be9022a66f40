"""The host half of OfflineVC / OfflineReflowVC (ddsp_svc_b200/offline.py) against goldens from the live reference
(tests/golden/make_golden_offline.py): the Slicer's silence state machine, main.py's split() and its assembly
bookkeeping, on seeded synthetic speech rebuilt here from its seed."""
import os

import numpy as np
import pytest

from ddsp_svc_b200 import offline
from tests import offline_oracle as oo

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "offline_slicer.npz"))
CASES = [(name, sr) for sr in oo.SLICER_RATES for name in sorted(oo.SLICER_CASES)]


def host_split(name, sr):
    audio = oo.slicer_case(name, sr)
    p = offline.SlicerParams(sr)
    tags = [] if audio.shape[0] <= p.min_length else offline.silence_tags(oo.rms64(audio, p.win, p.hop)[0], p)
    return audio, p, offline.slicer_chunks(tags, audio.shape[0], p.hop)


def test_slicer_params_are_the_reference_constructor():
    p = offline.SlicerParams(44100)
    assert (p.hop, p.win, p.min_length, p.min_interval, p.max_sil_kept) == (882, 3528, 250, 15, 250)
    p = offline.SlicerParams(16000)
    assert (p.hop, p.win, p.min_length, p.min_interval, p.max_sil_kept) == (320, 1280, 250, 15, 250)
    assert p.threshold == 10 ** (-40 / 20.)


@pytest.mark.parametrize("name,sr", CASES)
def test_rms_framing_matches_the_golden(name, sr):
    audio, p, _ = host_split(name, sr)
    rms = GOLD["%s_%d_rms" % (name, sr)]
    assert rms.shape == (1 + audio.shape[0] // p.hop,)
    assert np.array_equal(oo.rms64(audio, p.win, p.hop)[0], rms)


@pytest.mark.parametrize("name,sr", CASES)
def test_state_machine_reproduces_the_slicer(name, sr):
    _, _, chunks = host_split(name, sr)
    want = GOLD["%s_%d_chunks" % (name, sr)]
    assert np.array_equal(np.array([[b, e, int(s)] for b, e, s in chunks], dtype=np.int64).reshape(-1, 3), want)


def test_the_cases_cover_every_branch():
    """each case's silent run has the length its name says, in frames, against the Slicer's bounds"""
    for sr in oo.SLICER_RATES:
        p = offline.SlicerParams(sr)
        k = p.max_sil_kept

        def runs(name):
            audio = oo.slicer_case(name, sr)
            quiet = np.concatenate([[0], oo.rms64(audio, p.win, p.hop)[0] < np.float32(p.threshold), [0]]).astype(int)
            edges = np.flatnonzero(np.diff(quiet))
            return [(int(a), int(b - a)) for a, b in zip(edges[::2], edges[1::2])], quiet.shape[0] - 2
        (first, n), total = runs("leading_silence")[0][0], runs("leading_silence")[1]
        assert first == 0 and n > k
        (first, n), total = runs("trailing_silence")[0][-1], runs("trailing_silence")[1]
        assert first + n == total and n >= p.min_interval
        for name, lo, hi in (("gap_within_max_sil_kept", p.min_interval, k), ("gap_up_to_twice_max_sil_kept", k + 1, 2 * k),
                             ("gap_beyond_twice_max_sil_kept", 2 * k + 1, 10 ** 9), ("gap_below_min_interval", 1, p.min_interval - 1)):
            (first, n), = runs(name)[0]
            assert first >= p.min_length and lo <= n <= hi, (name, sr, first, n)
        assert runs("no_silence")[0] == []
        assert oo.slicer_case("under_min_length", sr).shape[0] <= p.min_length


def test_first_minimum_wins():
    p = offline.SlicerParams(44100)
    rms = np.full(600, 0.5, np.float32)
    rms[300:330] = 0.001                                            # 30 silent frames, all equal: argmin's first
    assert offline.silence_tags(rms, p) == [(300, 300)]


@pytest.mark.parametrize("name,sr", CASES)
def test_split_matches_main_py(name, sr):
    _, _, chunks = host_split(name, sr)
    got = offline.split_frames(chunks, oo.SPLIT_HOP[sr])
    assert np.array_equal(np.array(got, dtype=np.int64).reshape(-1, 2), GOLD["%s_%d_split" % (name, sr)])
    assert got == offline.split_frames(chunks, float(oo.SPLIT_HOP[sr]))       # main.py's hop_size is a float


ASSEMBLIES = sorted(k[:-5] for k in GOLD.files if k.endswith("_seed"))


@pytest.mark.parametrize("tag", ASSEMBLIES)
def test_assembly_bookkeeping_matches_main_py(tag):
    key = tag.split("_assembly")[0]
    frames = GOLD[key + "_split"]
    A = oo.ASSEMBLY
    segs = oo.assembly_segments(frames[:, 0], frames[:, 1], seed=int(GOLD[tag + "_seed"]),
                                short=len(frames) - 1 if tag.endswith("_short") else None, **A)
    if tag + "_error" in GOLD.files:                                  # numpy's cross_fade cannot broadcast
        with pytest.raises(ValueError, match="cross-fade"):
            offline.assembly_plan(frames[:, 0].tolist(), [s.shape[0] for s in segs], A["block_size"], A["out_sr"],
                                  A["model_sr"])
        return
    plan, total = offline.assembly_plan(frames[:, 0].tolist(), [s.shape[0] for s in segs], A["block_size"],
                                        A["out_sr"], A["model_sr"])
    want = GOLD[tag]
    assert total == want.shape[0]
    assert any(f > 0 for _, f in plan) == (len(frames) > 1)
    assert np.array_equal(oo.assemble64(segs, plan, total), want)


def test_assembly_plan_rounds_like_python():
    # 3 * 512 * 48000 / 44100 = 1671.836..., 5 * 512 * 48000 / 44100 = 2786.39...: round-half-even on exact halves too
    plan, total = offline.assembly_plan([0, 3, 5], [1700, 1200, 100], 512, 48000, 44100)
    assert plan == [(0, 0), (1672, 28), (2786, 86)] and total == 2886
    assert offline.assembly_plan([1], [5], 1, 3, 2) == ([(2, 0)], 7)           # round(1.5) = 2
    assert offline.assembly_plan([1], [5], 5, 1, 2) == ([(2, 0)], 7)           # round(2.5) = 2


def test_reflow_settings_follow_main_reflow():
    from ddsp_svc_b200.dropin import DotDict
    args = DotDict({"model": {"t_start": 0.5}, "infer": {"method": "rk4", "infer_step": 3}})
    assert offline.reflow_settings(args) == (3, "rk4", 0.5)
    assert offline.reflow_settings(args, 2, "euler", 0.2) == (2, "euler", 0.5)  # raised to the model's floor
    assert offline.reflow_settings(args, 0, "euler", 0.8) == (0, "euler", 0.8)
    assert offline.reflow_settings(DotDict({"model": {}}), 2, "euler", "auto") == (2, "euler", 0.0)
    with pytest.raises(ValueError, match="negative"):
        offline.reflow_settings(args, -1)
    with pytest.raises(ValueError, match="infer.method"):
        offline.reflow_settings(DotDict({"model": {}}), 2, "auto")


def test_constructor_errors_come_before_loading():
    with pytest.raises(ValueError, match="CUDA device"):
        offline.OfflineVC("no/such/model.pt", device="cpu")
    with pytest.raises(ValueError, match="CUDA device"):
        offline.OfflineReflowVC("no/such/model.pt", device="cpu")
    with pytest.raises(ValueError, match="'rmvpe' only"):
        offline.OfflineVC("no/such/model.pt", pitch_extractor="harvest")
    with pytest.raises(ValueError, match="'rmvpe' only"):
        offline.OfflineReflowVC("no/such/model.pt", pitch_extractor="crepe")
