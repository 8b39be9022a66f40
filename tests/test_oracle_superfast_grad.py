"""The gradient oracles of CombSubSuperFast against the reference's own autograd gradient (CPU).

tests/golden/superfast_grad_*.npz hold dense.grad of the live reference (make_golden_superfast_grad.py).
* oracle.torch_port.superfast_forward under autograd runs the reference's ATen operators, so its gradient must be
  bit-identical; that licenses the port as the gradient oracle for shapes too large for goldens;
* tests/superfast_grad_closed_form.superfast_grad restates the backward in float64 and must sit at the fp32 floor of
  it."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import synthetic as syn
from oracle import torch_port as tp
from tests import superfast_grad_closed_form as cfg
from tests import util
from tests.golden import make_golden_superfast_grad as GG

NAMES = list(GG.CASES)
N_BINS = GG.WIN // 2 + 1


def load(name):
    inp = GG.build_inputs(name)
    z = np.load(GG.path(name), allow_pickle=False)
    gold = {k: z[k] for k in z.files}
    for k, v in GG.input_checksums(inp).items():
        assert abs(float(gold[k]) - v) <= 1e-9 * max(1.0, abs(v)), "input %s of %s differs from the golden's" % (k, name)
    return inp, gold


def rel_rms(got, ref):
    return util.rms(np.asarray(got, np.float64) - ref) / util.rms(ref)


@pytest.mark.parametrize("name", NAMES)
def test_port_autograd_is_bit_identical_to_reference(name):
    inp, gold = load(name)
    dense = inp["dense"].clone().requires_grad_(True)
    out = tp.superfast_forward(inp["f0"], syn.split_views(dense, GG.split_map()), GG.SR, GG.P, GG.WIN,
                               noise=inp["noise"])
    assert torch.equal(out["signal"].detach(), torch.from_numpy(gold["signal"]))
    (out["signal"] * inp["cot"]).sum().backward()
    assert torch.equal(dense.grad, torch.from_numpy(gold["grad"]))


@pytest.mark.parametrize("name", NAMES)
def test_closed_form_gradient_matches_reference(name):
    inp, gold = load(name)
    got = cfg.superfast_grad(inp["f0"].numpy(), {k: v.numpy() for k, v in inp["ctrls"].items()}, GG.SR, GG.P, GG.WIN,
                             inp["noise"].numpy(), inp["cot"].numpy())
    for i, key in enumerate(GG.split_map()):
        ref = gold["grad"][..., i * N_BINS:(i + 1) * N_BINS].astype(np.float64)
        assert got[key].shape == ref.shape
        e = rel_rms(got[key], ref)
        assert e <= 1e-6, (name, key, e)
