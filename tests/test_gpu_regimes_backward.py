"""GPU: the CUDA backwards of Sins, CombSub, CombSubFast and CombSubSuperFast at the input regimes of tests/regimes.py
(the pairing of tests/test_gpu_regimes_forward.py).  The backwards multiply by the activations' derivatives -- exp(c),
pi (1 - tanh^2 c), j pi H -- so saturated and very negative controls are where a gradient that should be ~0 or ~1e3
shows whether it was computed or is merely small.

Every output the op returns carries a cotangent (signal, and harmonic / noise for Sins and CombSub).  Truth is the
float64 closed form (tests/*_grad_closed_form.py) at the exact float64 source; ref32 is torch autograd through
oracle.torch_port in fp32, training phase.  Per control group and per utterance row -- the groups' scales differ by 1e6
in these regimes, the rows' by 1e10 in mixed_rows --

    |gpu - truth| / |truth| <= max(1e-5, FACTOR x |ref32 - truth| / |truth|)          (L2 norms)

and where a group's true gradient is below 1e-12 of the row's largest group, |gpu - truth| <= 1e-12 x that largest
norm instead.  The errors go to tests.report."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import ops, synthetic as syn
from tests import regimes as R
from tests import report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P, WIN = R.SR, R.P, R.WIN
FACTOR = 2.0


def gpu_grad(inp, only=None, rows=None):
    """{control: numpy [B, nF, C]} of R.objective through the kernels (training phase); ``rows``: a slice of the batch"""
    s = inp["synth"]
    if rows is not None:
        inp = dict(inp, **{k: inp[k][rows] for k in ("f0", "dense", "noise", "cot", "cot_h", "cot_n") if k in inp})
    f0 = inp["f0"].to(DEV)
    leaf = inp["dense"].to(DEV).requires_grad_(True)
    c = syn.split_views(leaf, R.SPLITS[s])
    nz = inp["noise"].to(DEV)
    if s == "superfast":
        ws, _ = ops.superfast_scan(f0, P, SR)
        out = (ops.superfast_synth(ws, c["harmonic_magnitude"], c["harmonic_phase"], c["noise_magnitude"],
                                   c["noise_phase"], P, WIN, noise_in=nz),)
    else:
        fph, _ = ops.phase_scan(f0, P, SR, infer=False)
        if s == "sins":
            out = ops.sins_synth(f0, fph, c["amplitudes"], c["group_delay"], c["noise_magnitude"], P, SR, noise_in=nz,
                                 infer=False)
        elif s == "combsub":
            out = ops.combsub_synth(f0, fph, c["group_delay"], c["harmonic_magnitude"], c["noise_magnitude"], P, SR,
                                    noise_in=nz, infer=False)
        else:
            comb = ops.comb_source(f0, fph, P, SR, infer=False)
            out = (ops.combsubfast_filter(comb, c["harmonic_magnitude"], c["harmonic_phase"], c["noise_magnitude"], P,
                                          noise_in=nz),)
    R.objective(dict(zip(R.outputs_of(s), out)), inp, only).backward()
    assert torch.isfinite(leaf.grad).all()
    return {k: v.cpu().numpy() for k, v in syn.split_views(leaf.grad, R.SPLITS[s]).items()}


def check(tag, got, ref32, truth):
    errs = R.grad_errors(got, ref32, truth)
    bad = []
    for k, e in errs.items():
        bound = R.grad_bound(e, FACTOR)
        report.record("regimes_backward/%s_%s" % (tag, k), gpu_vs_truth=e["got"].max(), ref32_vs_truth=e["ref"].max(),
                      ratio=(e["got"] / bound).max(), norm_min=e["norm"].min(), norm_max=e["norm"].max(),
                      relative=bool(e["relative"].all()))
        for b in np.nonzero(~(e["got"] <= bound))[0]:
            bad.append((k, int(b), e["got"][b], bound[b]))
    assert not bad, (tag, bad)


@pytest.mark.parametrize("case", R.TABLE, ids=R.CASE_IDS)
@pytest.mark.parametrize("synth", list(R.SPLITS))
def test_gradient_at_regime(synth, case):
    inp = R.build(synth, *case, with_cotangents=True)
    check("%s_%s" % (synth, "-".join(case)), gpu_grad(inp), R.port_grad(inp), R.truth_grad(inp))


@pytest.mark.parametrize("only", ["harmonic", "noise"])
@pytest.mark.parametrize("synth", R.HAS_PARTS)
def test_gradient_of_one_part_alone(synth, only):
    """a cotangent on the harmonic (noise) output alone: the other side's controls get exactly zero, not something
    small, and the rest stays within the criterion"""
    inp = R.build(synth, "octave_jumps", "saturated_gd", with_cotangents=True)
    got, truth = gpu_grad(inp, only), R.truth_grad(inp, only)
    dead = ["noise_magnitude"] if only == "harmonic" else [k for k in truth if k != "noise_magnitude"]
    for k in dead:
        assert not truth[k].any() and not got[k].any(), (synth, only, k)
    live = lambda d: {k: v for k, v in d.items() if k not in dead}
    check("%s_%s_only" % (synth, only), live(got), live(R.port_grad(inp, only)), live(truth))


@pytest.mark.parametrize("pitch", ["onsets", "near_zero"])
@pytest.mark.parametrize("synth", list(R.SPLITS))
def test_cold_row_does_not_feel_the_hot_row(synth, pitch):
    """mixed_rows: row 0 (every magnitude -20, gradients ~1e-9) next to row 1 (+4, gradients ~1e3).  Row 0's gradient
    computed in the batch equals, bit for bit, row 0's gradient computed alone."""
    inp = R.build(synth, pitch, "mixed_rows", with_cotangents=True)
    both, alone = gpu_grad(inp), gpu_grad(inp, rows=slice(0, 1))
    for k in both:
        assert np.array_equal(both[k][:1], alone[k]), (synth, pitch, k, np.abs(both[k][:1] - alone[k]).max())
    k = "noise_magnitude"                       # present in every split, and never zero (the noise is always on)
    assert 0 < np.abs(both[k][0]).max() < 1e-6 * np.abs(both[k][1]).max()
