"""OfflineDiffVC's host half (ddsp_svc_b200/offline.py): ``diff_settings`` against main_diff.py's and batch_infer.py's
own selection lines (tests/golden/make_golden_offline_diff.py) over every model type, k_step, DDSP checkpoint, sampler
setting and diffusion speaker; its ValueErrors; and the comparison it shares with DiffGtMel.check_args."""
import json
import os

import pytest

from ddsp_svc_b200 import diffusion_vocoder, offline
from ddsp_svc_b200.dropin import DotDict

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "offline_diff_settings.json")))
CASES = GOLD["cases"]


def configs(case):
    args = DotDict({"data": dict(GOLD["data"]), "infer": dict(GOLD["infer"]),
                    "model": {"type": case["model_type"], "k_step_max": GOLD["k_step_max"]}})
    ddsp = case["ddsp"]
    if ddsp == "none":
        return args, None
    data = dict(GOLD["data"])
    if ddsp != "compatible":
        data[ddsp] = GOLD["bad"][ddsp]
    return args, DotDict({"data": data})


def case_id(c):
    return "%s-k%s-%s-%s-%s-spk%s-%s" % (c["model_type"], c["k_step"], c["ddsp"], c["speedup"], c["method"],
                                         c["diff_spk_id"], "whole" if c["whole"] else "sliced")


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_diff_settings_match_the_drivers(case):
    args, ddsp_args = configs(case)
    s = offline.diff_settings(args, ddsp_args, case["k_step"], case["speedup"], case["method"], case["diff_spk_id"],
                              case["whole"])
    want = case["want"]
    mode = "ddsp" if want["ddsp"] else "input_mel" if want["input_mel"] else "none"
    assert s.mode == mode
    assert s.k_step == want["k_step"]
    assert s.infer_speedup == want["infer_speedup"] and s.method == want["method"]
    assert (GOLD["spk_id"] if s.diff_spk_id is None else s.diff_spk_id) == want["diff_spk_id"]


def test_the_grid_reaches_every_mode_of_each_driver():
    seen = {(c["model_type"], c["whole"], c["want"]["ddsp"], c["want"]["input_mel"]) for c in CASES}
    for kind in ("Diffusion", "DiffusionNew", "DiffusionFast"):
        for whole in (False, True):
            assert (kind, whole, True, False) in seen and (kind, whole, False, False) in seen
            assert ((kind, whole, False, True) in seen) == (kind == "Diffusion")


def test_auto_needs_the_infer_section():
    args = DotDict({"data": dict(GOLD["data"]), "model": {"type": "DiffusionNew", "k_step_max": 100},
                    "infer": {"method": "ddim"}})
    with pytest.raises(ValueError, match="infer.speedup"):
        offline.diff_settings(args, None)
    assert offline.diff_settings(args, None, speedup=5).method == "ddim"
    del args["infer"]
    with pytest.raises(ValueError, match="infer.method"):
        offline.diff_settings(args, None, speedup=5)
    with pytest.raises(ValueError, match="Unknown Model"):
        offline.diff_settings(DotDict({"model": {"type": "Reflow"}}), None, speedup=5, method="ddim")


def test_one_comparison_for_both_checks():
    a = DotDict({"data": dict(GOLD["data"])})
    b = DotDict({"data": dict(GOLD["data"], block_size=256, encoder="hubertsoft")})
    assert diffusion_vocoder.data_mismatches(a, a) == []
    assert diffusion_vocoder.data_mismatches(a, b) == ["block_size", "encoder"]
    g = diffusion_vocoder.DiffGtMel()
    assert g.check_args(a, a) is True
    # DiffGtMel raises for the first mismatch in infer_gt_mel.py's order: block_size, sampling_rate, encoder
    c = DotDict({"data": dict(GOLD["data"], sampling_rate=48000, block_size=256)})
    with pytest.raises(ValueError, match="^the DDSP and diffusion models' block_size differ$"):
        g.check_args(a, c)
    with pytest.raises(ValueError, match="^the DDSP and diffusion models' sampling_rate differ$"):
        g.check_args(a, DotDict({"data": dict(GOLD["data"], sampling_rate=48000, encoder="x")}))
    with pytest.raises(ValueError, match="^the DDSP and diffusion models' encoder differ$"):
        g.check_args(a, DotDict({"data": dict(GOLD["data"], encoder="x")}))


def test_constructor_errors_come_before_loading():
    with pytest.raises(ValueError, match="CUDA device"):
        offline.OfflineDiffVC("no/such/model.pt", device="cpu")
    with pytest.raises(ValueError, match="'rmvpe' only"):
        offline.OfflineDiffVC("no/such/model.pt", pitch_extractor="crepe")
