"""The gradient oracles of CombSubFast (training phase) against the reference's own autograd gradient (CPU).

tests/golden/csfast_grad_*.npz hold dense.grad of the live reference (make_golden_combsubfast_grad.py).
* oracle.torch_port.combsubfast_forward(..., infer=False) under autograd runs the reference's ATen operators, so its
  gradient must be bit-identical; that licenses the port as the gradient oracle for shapes too large for goldens;
* tests/combsubfast_grad_closed_form.combsubfast_grad restates the backward in float64 and, fed the comb the
  reference filtered (the port's "comb"), must sit at the fp32 floor of it."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import synthetic as syn
from oracle import ref_loader
from oracle import torch_port as tp
from tests import combsubfast_grad_closed_form as cfg
from tests import util
from tests.golden import make_golden_combsubfast_grad as GG

NAMES = list(GG.CASES)
NB = GG.NB


def load(name):
    inp = GG.build_inputs(name)
    z = np.load(GG.path(name), allow_pickle=False)
    gold = {k: z[k] for k in z.files}
    for k, v in GG.input_checksums(inp).items():
        assert abs(float(gold[k]) - v) <= 1e-9 * max(1.0, abs(v)), "input %s of %s differs from the golden's" % (k, name)
    return inp, gold


def rel_rms(got, ref):
    return util.rms(np.asarray(got, np.float64) - ref) / util.rms(ref)


def port(inp, dense):
    return tp.combsubfast_forward(inp["f0"], syn.split_views(dense, GG.split_map()), GG.SR, GG.P, noise=inp["noise"],
                                  initial_phase=inp["initial_phase"], infer=False)


@pytest.mark.parametrize("name", NAMES)
def test_port_autograd_is_bit_identical_to_reference(name):
    """Bit for bit against the reference's own signal and gradient computed on the same FFT code path.  torch's CPU
    FFT (MKL) dispatches on the instruction set and its paths differ in the last bits, so the reference itself
    computes other bits on another path: the stored golden is the reference's result where this machine's FFT
    fingerprint equals the one stored with it; elsewhere the live reference is run in this process.  Against the
    stored golden the port must sit at the fp32 floor on every path."""
    inp, gold = load(name)
    dense = inp["dense"].clone().requires_grad_(True)
    out = port(inp, dense)
    (out["signal"] * inp["cot"]).sum().backward()
    got = {"signal": out["signal"].detach(), "grad": dense.grad}
    for key, v in got.items():
        e = rel_rms(v.numpy(), gold[key].astype(np.float64))
        assert e <= 1e-6, (name, key, e)
    if str(gold["fft_fingerprint"]) == GG.fft_fingerprint():
        ref = {k: torch.from_numpy(gold[k]) for k in got}
    elif ref_loader.available():
        ref = GG.run_reference(name)[1]
    else:
        pytest.skip("this machine's FFT code path differs from the goldens' and the live reference is not available")
    for key, v in got.items():
        assert torch.equal(v, ref[key]), (name, key)


@pytest.mark.parametrize("name", NAMES)
def test_closed_form_gradient_matches_reference(name):
    inp, gold = load(name)
    with torch.no_grad():
        comb = port(inp, inp["dense"])["comb"].numpy()
    got = cfg.combsubfast_grad(comb, {k: v.numpy() for k, v in inp["ctrls"].items()}, GG.P, inp["noise"].numpy(),
                               inp["cot"].numpy())
    for i, key in enumerate(GG.split_map()):
        ref = gold["grad"][..., i * NB:(i + 1) * NB].astype(np.float64)
        assert got[key].shape == ref.shape
        e = util.rms(got[key] - ref) / util.rms(ref)
        assert e <= 1e-6, (name, key, e)
