"""The float64 plain-torch oracle of the reflow loss (tests/reflow_oracle.VelocityNet + make_golden_reflow_grad.oracle_loss)
against the reference's own loss and gradients stored by tests/golden/make_golden_reflow_grad.py, on the CPU.  This pins
the oracle the GPU tests use where the reference does not exist (the 512-wide network at the training batch)."""
import json

import numpy as np
import pytest
import torch

from tests.golden import make_golden_reflow as mk
from tests.golden import make_golden_reflow_grad as GR


def oracle_gradients(name):
    d = np.load(GR.path(name))
    net = mk.build_oracle(GR.MODEL).double()
    cond = torch.from_numpy(d["condition"]).double().requires_grad_(True)
    loss = GR.oracle_loss(net, cond, torch.from_numpy(d["gt_spec"]), torch.from_numpy(d["t"]), torch.from_numpy(d["x0"]))
    loss.backward()
    grads = {n: p.grad for n, p in net.named_parameters()}
    grads["condition"] = cond.grad
    return d, loss, grads


@pytest.mark.parametrize("name", list(GR.CASES))
def test_oracle_reproduces_the_references_loss_and_gradients(name):
    d, loss, grads = oracle_gradients(name)
    assert abs(loss.item() - float(d["loss64"])) <= 1e-12 * abs(float(d["loss64"]))
    assert {n for n, g in grads.items() if g is None} == set(json.loads(str(d["none"])))
    kept = GR.stored(name, grads)
    assert set(kept) == {k[4:] for k in d.files if k.startswith("f64/")}
    for n, g in kept.items():
        want = d["f64/" + n].astype(np.float64)
        # the stored gradient is the float64 one rounded to fp32: 2^-24 relative per entry
        assert np.abs(g.numpy() - want).max() <= 1e-7 * np.abs(want).max() + 1e-300, n
        assert float(d["err32/" + n]) < 1e-3, n                  # the reference's own fp32 run is fp32-grade


def test_the_fixtures_are_not_degenerate():
    """every gradient is non-zero (the seeded output projection), the bounds case clips t and its fp32 weights at the
    bounds underflow to 0, the short case is shorter than the convolution's reach"""
    for name, c in GR.CASES.items():
        d = np.load(GR.path(name))
        assert all(np.abs(d[k]).max() > 0 for k in d.files if k.startswith("f64/")), name
        assert (d["t"] >= np.float32(1e-7)).all() and (d["t"] <= np.float32(1 - 1e-7)).all()
    d = np.load(GR.path("reflow_grad_w128_b3_t24_bounds"))
    assert d["t"][0] == np.float32(1e-7) and d["t"][2] == np.float32(1 - 1e-7)
    t = torch.from_numpy(d["t"])
    w = 0.398942 / t / (1 - t) * torch.exp(-0.5 * torch.log(t / (1 - t)) ** 2)
    assert w[0] == 0 and w[2] == 0 and w[1] > 0
    assert GR.CASES["reflow_grad_w128_b1_t9_t07"]["T"] < 31


def test_seeded_draws_follow_the_references_order():
    """t = t_start + (1 - t_start) rand(B), clipped, then x_0 = randn_like of the transposed [B, 1, M, T] view, which
    keeps that view's strides: the same numbers as an empty_strided draw with those strides, and neither randn(B, 1, M, T)
    nor randn(B, T, M)"""
    B, T, M = 2, 7, 5
    torch.manual_seed(3)
    t, x0 = GR.draws(B, T, M, 0.7)
    torch.manual_seed(3)
    x1 = torch.zeros(B, T, M).transpose(1, 2)[:, None]
    t_ref = torch.clip(0.7 + 0.3 * torch.rand(B), 1e-7, 1 - 1e-7)
    x0_ref = torch.randn_like(x1)
    assert torch.equal(t, t_ref) and torch.equal(x0, x0_ref[:, 0].transpose(1, 2))
    for shape in ((B, 1, M, T), (B, T, M)):
        torch.manual_seed(3)
        torch.rand(B)
        other = torch.randn(shape)
        assert not torch.equal(x0, other.reshape(B, M, T).transpose(1, 2) if len(shape) == 4 else other)
