"""The gradient oracles of the old CombSub (training phase) against the reference's own autograd gradient (CPU).

tests/golden/combsub_grad_*.npz hold dense.grad of the live reference (make_golden_combsub_grad.py).
* oracle.torch_port.combsub_forward(infer=False) under autograd runs the reference's ATen operators, so its gradient
  must be bit-identical; that licenses the port as the gradient oracle for shapes too large for goldens;
* tests/combsub_grad_closed_form.combsub_grad restates the backward in float64: fed the same comb, it must match
  float64 autograd of the port to ~1e-11, and the goldens (fed the reference's comb) at the fp32 floor."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import synthetic as syn
from oracle import torch_port as tp
from tests import combsub_grad_closed_form as cfg
from tests import util
from tests.golden import make_golden_combsub_grad as GG

NAMES = list(GG.CASES)
KEYS = ("group_delay", "harmonic_magnitude", "noise_magnitude")


def load(name):
    inp = GG.build_inputs(name)
    inp["name"] = name
    z = np.load(GG.path(name), allow_pickle=False)
    gold = {k: z[k] for k in z.files}
    for k, v in GG.input_checksums(inp).items():
        assert abs(float(gold[k]) - v) <= 1e-9 * max(1.0, abs(v)), "input %s of %s differs from the golden's" % (k, name)
    return inp, gold


def split_grad(name, dense_grad):
    return {k: np.asarray(v, np.float64) for k, v in
            syn.split_views(torch.as_tensor(np.asarray(dense_grad)), GG.split_map(name)).items()}


def rel_rms(got, ref):
    return util.rms(np.asarray(got, np.float64) - ref) / util.rms(ref)


def port(inp, dense, dtype=torch.float32):
    return tp.combsub_forward(inp["f0"].to(dtype), syn.split_views(dense, GG.split_map(inp["name"])), GG.SR, GG.P,
                              noise=inp["noise"].to(dtype), infer=False)


def reference_comb(inp):
    """the comb the reference filters (its fp32 training-phase phase), [B, T]"""
    with torch.no_grad():
        return port(inp, inp["dense"])["comb"].numpy()


def closed_form(inp, comb, allpassed_in=None):
    opt = lambda k: None if inp[k] is None else inp[k].numpy()
    return cfg.combsub_grad(inp["f0"].numpy(), {k: v.numpy() for k, v in inp["ctrls"].items()}, comb, GG.SR, GG.P,
                            inp["noise"].numpy(), inp["cot"].numpy(), opt("cot_h"), opt("cot_n"), allpassed_in)


def error_model(name, inp, gold_grad, comb):
    """-> (truth {control: float64 [B, nF, C]} at ``comb``, {control: bound against truth}, {control: bound against
    the golden}).  The first bound is the fp32 reference's own relative RMS error against float64 at ITS comb (times
    ``RATIO``, not below ``FLOOR``); the second adds twice the relative distance between the float64 gradients at the
    reference's comb and at ``comb`` (the comb source differs, not the backward: tests/test_emu_combsub_backward.py,
    tests/test_gpu_combsub_backward.py)."""
    at_ref = closed_form(inp, reference_comb(inp))
    gold = split_grad(name, gold_grad)
    truth = closed_form(inp, comb)
    tight = {k: max(RATIO * rel_rms(gold[k], at_ref[k]), FLOOR[k]) for k in KEYS}
    return truth, tight, {k: tight[k] + 2 * rel_rms(at_ref[k], truth[k]) for k in KEYS}


# a kernel's relative RMS error against float64 at its own comb: RATIO x the fp32 reference's own error, and not below
# the random-rounding floor of one fp32 sum of 2P products -- for the all-pass control, of the cascade's sums in a row
# (da sums up to 2 x 1024 products per sample through the forward's fp32 harmonic impulse response, then dh_ap 2P)
RATIO = 3.0
FLOOR = {"group_delay": 2.0 ** -24 * np.sqrt(2 * GG.P + 4 * 1024), "harmonic_magnitude": 2.0 ** -24 * np.sqrt(2 * GG.P),
         "noise_magnitude": 2.0 ** -24 * np.sqrt(2 * GG.P)}


@pytest.mark.parametrize("name", NAMES)
def test_port_autograd_is_bit_identical_to_reference(name):
    inp, gold = load(name)
    dense = inp["dense"].clone().requires_grad_(True)
    out = port(inp, dense)
    assert torch.equal(out["signal"].detach(), torch.from_numpy(gold["signal"]))
    GG.objective(out["signal"], out["harmonic"], out["noise"], inp).backward()
    assert torch.equal(dense.grad, torch.from_numpy(gold["grad"]))


@pytest.mark.parametrize("name", NAMES)
def test_closed_form_matches_float64_autograd(name):
    """the port's operators in float64 under autograd, and the closed form fed the same (float64) comb.  The port's
    Hann window is torch.hann_window's fp32 table, which bounds the noise control at the fp32 level."""
    inp, _ = load(name)
    dense = inp["dense"].double().requires_grad_(True)
    out = port(inp, dense, torch.float64)
    d = {k: (None if inp[k] is None else inp[k].double()) for k in ("cot", "cot_h", "cot_n")}
    GG.objective(out["signal"], out["harmonic"], out["noise"], d).backward()
    want = split_grad(name, dense.grad.numpy())
    got = closed_form(inp, out["comb"].detach().numpy())
    for k in KEYS:
        e = rel_rms(got[k], want[k])
        assert e <= (2e-7 if k == "noise_magnitude" else 1e-10), (name, k, e)


@pytest.mark.parametrize("name", NAMES)
def test_closed_form_gradient_matches_reference(name):
    """fp32 floor: the reference's fp32 FFTs and sums against float64 at the reference's own comb"""
    inp, gold = load(name)
    got = closed_form(inp, reference_comb(inp))
    ref = split_grad(name, gold["grad"])
    for k in KEYS:
        assert got[k].shape == ref[k].shape
        e = rel_rms(got[k], ref[k])
        assert e <= 5e-5, (name, k, e)
