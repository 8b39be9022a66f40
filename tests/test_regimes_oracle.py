"""CPU: the input regimes of tests/regimes.py are what they say, and the budget the GPU regime tests lean on -- the
distance of the reference's own fp32 arithmetic (oracle.torch_port) from the float64 closed form -- is finite, recorded
and pinned for every table entry, so a change to either oracle that inflates it is seen here."""
import numpy as np
import pytest
import torch

from tests import regimes as R
from tests import report

# the fp32 reference's RMS distance from float64 per synthesizer, relative to max(signal RMS, 0.01), worst table entry
# and worst row: measured 4.1e-4 (sins), 9.5e-4 (combsub), 9.4e-4 (combsubfast), all in the training phase (fp32
# cumsum of the phase), and 2.6e-4 (superfast); 1.8e-5 / 1.8e-5 / 6.2e-6 with infer=True.  Pinned with 4x headroom.
PINNED = {("sins", False): 1.7e-3, ("combsub", False): 4e-3, ("combsubfast", False): 4e-3,
          ("sins", True): 8e-5, ("combsub", True): 8e-5, ("combsubfast", True): 3e-5, ("superfast", True): 1e-3}


@pytest.mark.parametrize("name", list(R.PITCH))
@pytest.mark.parametrize("shape", [(3, 48), (2, 24), (3, 200)])
def test_pitch_regime_is_what_it_says(name, shape):
    B, nF = shape
    if name == "onsets" and B < 3:
        pytest.skip("the onsets regime needs three rows")
    for seed in (0, 1, 12345):
        f0 = R.PITCH[name](B, nF, seed)
        assert f0.shape == (B, nF, 1)
        R.check_pitch(name, f0)
        assert torch.equal(f0, R.PITCH[name](B, nF, seed))              # seeded


@pytest.mark.parametrize("name", list(R.CTRL))
@pytest.mark.parametrize("synth", list(R.SPLITS))
def test_control_regime_is_what_it_says(name, synth):
    split = R.SPLITS[synth]
    for seed in (0, 7):
        dense, views = R.CTRL[name](2, 24, split, seed)
        assert dense.shape == (2, 24, sum(split.values())) and list(views) == list(split)
        R.check_ctrl(name, views)
        assert torch.equal(dense, R.CTRL[name](2, 24, split, seed)[0])


def test_table_pairs_every_regime_with_every_synthesizer():
    assert {p for p, _ in R.TABLE} == set(R.PITCH) and {c for _, c in R.TABLE} == set(R.CTRL)
    assert len(set(R.TABLE)) == len(R.TABLE)
    for synth in R.SPLITS:
        for p, c in R.TABLE:
            inp = R.build(synth, p, c)
            R.check_pitch(p, inp["f0"])
            R.check_ctrl(c, inp["ctrls"])


@pytest.mark.parametrize("case", R.TABLE, ids=R.CASE_IDS)
@pytest.mark.parametrize("synth,infer", [(s, i) for s in R.SPLITS for i in ((True, False) if s in R.HAS_INFER else (True,))])
def test_fp32_reference_against_float64(synth, infer, case):
    inp = R.build(synth, *case)
    truth = R.truth_forward(inp)
    with torch.no_grad():
        ref = R.port_forward(inp, infer=infer)
    for key in R.outputs_of(synth):
        assert np.isfinite(truth[key]).all() and torch.isfinite(ref[key]).all()
        e = R.forward_errors(ref[key].numpy(), ref[key].numpy(), truth[key])
        rel = float(np.max(e["ref_rms"] / np.maximum(e["truth_rms"], 0.01)))
        report.record("regimes_oracle/%s_%s_%s_%s" % (synth, "infer" if infer else "train", "-".join(case), key),
                      ref32_vs_truth=e["ref_rms"].max(), floor=e["floor"].min(), truth_rms=e["truth_rms"].max(), rel=rel)
        assert rel <= PINNED[synth, infer], (synth, infer, case, key, rel)
    if synth in R.HAS_PARTS:
        assert np.allclose(truth["signal"], truth["harmonic"] + truth["noise"], rtol=0, atol=1e-12 * np.abs(truth["signal"]).max())
