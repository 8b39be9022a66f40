"""BatchedRealtimeVC's host logic without a GPU: the session settings and their defaults, the packing of the settings
into the per-row arrays the kernels read (at the precision of the single-session kernels' scalar arguments), the speaker
mix row, and the argument checks that run before any model is loaded."""
import ctypes

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import frontend
from ddsp_svc_b200.realtime import SESSION_DEFAULTS, BatchedRealtimeVC, RealtimeVC, session_rows, session_settings
from ddsp_svc_b200.unit2control import spk_mix_embedding


def test_defaults_are_realtimevc_defaults():
    import inspect
    params = inspect.signature(RealtimeVC.__init__).parameters
    for k, v in SESSION_DEFAULTS.items():
        assert params[k].default == v, k


def test_settings_merge_and_reject():
    assert session_settings({}) == SESSION_DEFAULTS
    c = session_settings(dict(spk_id=3, pitch_adjust=2.5))
    assert c["spk_id"] == 3 and c["pitch_adjust"] == 2.5 and c["threhold"] == SESSION_DEFAULTS["threhold"]
    assert session_settings(dict(threhold=-20), c)["spk_id"] == 3                   # update() keeps the rest
    with pytest.raises(ValueError, match="unknown"):
        session_settings(dict(key=3))
    with pytest.raises(ValueError, match="spk_mix_dict"):
        session_settings(dict(use_spk_mix=True))


def test_rows_at_scalar_argument_precision():
    pitches, dbs = [0.0, 5.0, -7.3, 12.0], [-45, -30.5, -60, 0]
    rows = session_rows([session_settings(dict(pitch_adjust=p, threhold=d, spk_id=i + 1))
                         for i, (p, d) in enumerate(zip(pitches, dbs))])
    assert rows["pitch_factor"].dtype == np.float32 and rows["threshold"].dtype == np.float32
    for i, (p, d) in enumerate(zip(pitches, dbs)):
        # RealtimeVC hands 2 ** (p / 12) and volume_mask's threshold to float parameters of the C ABI
        assert rows["pitch_factor"][i] == ctypes.c_float(2 ** (p / 12)).value
        assert rows["threshold"][i] == ctypes.c_float(frontend.mask_threshold(d)).value
    assert rows["spk_id"].tolist() == [1, 2, 3, 4] and rows["spk_id"].dtype == np.int64
    assert rows["spk_mix"] == [None] * 4


def test_mix_rows_only_with_use_spk_mix():
    mix = {1: 0.25, 2: 0.75}
    rows = session_rows([session_settings(dict(spk_mix_dict=mix)),
                         session_settings(dict(use_spk_mix=True, spk_mix_dict=mix))])
    assert rows["spk_mix"] == [None, mix]


def test_spk_mix_embedding_is_the_weighted_sum_in_dict_order():
    w = torch.randn(4, 256)
    got = spk_mix_embedding(w, {3: 0.5, "1": 0.25, 2: 0.25})
    want = 0 + 0.5 * w[2] + 0.25 * w[0] + 0.25 * w[1]
    assert torch.equal(got, want)


@pytest.mark.parametrize("kw,match", [(dict(enhancer_adaptive_key="auto"), "own"),
                                      (dict(sessions=[]), "at least one"),
                                      (dict(device="cpu"), "CUDA"),
                                      (dict(sessions=[dict(pitch=1)]), "unknown")])
def test_arguments_checked_before_loading(kw, match):
    args = dict(model_path="no/such/model.pt", sessions=[{}])
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        BatchedRealtimeVC(**args)
