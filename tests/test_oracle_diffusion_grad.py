"""The float64 restatement of the diffusion training loss (tests/diffusion_grad_oracle.py around tests/diffusion_oracle.
WaveNet and tests/reflow_oracle.VelocityNet) against the reference's own loss and gradients
(tests/golden/diffusion_grad_*.npz from tests/golden/make_golden_diffusion_grad.py), on the CPU.  The GPU tests measure the
kernels against this oracle where the reference does not exist, and replay the same fixtures
(tests/test_gpu_diffusion_backward.py)."""
import json

import numpy as np
import pytest
import torch

from tests import diffusion_grad_oracle as DG
from tests.golden import make_golden_diffusion as mk
from tests.golden import make_golden_diffusion_grad as GD


def _oracle(name, d):
    net = mk.build_oracle(GD.CASES[name]["model"]).double()
    c = torch.from_numpy(d["condition"]).double().requires_grad_(True)
    loss = DG.oracle_loss(net, c, torch.from_numpy(d["gt_spec"]), torch.from_numpy(d["t"]), torch.from_numpy(d["noise"]))
    loss.backward()
    grads = {n: p.grad for n, p in net.named_parameters()}
    grads["condition"] = c.grad
    return loss, grads


@pytest.mark.parametrize("name", list(GD.CASES))
def test_oracle_reproduces_the_references_loss_and_gradients(name):
    d = np.load(GD.path(name))
    loss, grads = _oracle(name, d)
    assert abs(loss.item() - float(d["loss64"])) <= 1e-12 * float(d["loss64"])
    assert abs(float(d["loss32"]) - float(d["loss64"])) <= 1e-5 * float(d["loss64"])
    assert {n for n, g in grads.items() if g is None} == set(json.loads(str(d["none"])))
    kept = GD.stored(name, grads)
    assert set(kept) == {k[4:] for k in d.files if k.startswith("f64/")}
    for n, g in kept.items():
        want = d["f64/" + n].astype(np.float64)
        err = np.sqrt(((g.numpy() - want) ** 2).mean()) / np.sqrt((want ** 2).mean())
        assert err <= 1e-6, (n, err)                               # the fixture holds fp32-rounded float64 values


@pytest.mark.parametrize("name", list(GD.CASES))
def test_fixtures_are_not_degenerate(name):
    """every stored gradient is non-zero and finite, every layer is reached, the loss is of order one, the steps are in
    range and the reference's own fp32 gradients are close to float64 but not identical"""
    d = np.load(GD.path(name))
    c = GD.CASES[name]
    assert 0.05 < float(d["loss64"]) < 50
    t = d["t"]
    assert t.dtype == np.int64 and t.shape == (c["B"],) and (t >= 0).all() and (t < 1000).all()
    if "t" in c:
        assert t.tolist() == c["t"]
    else:
        assert (t < GD.t_max(name)).all() and int(d["t_max"]) == GD.t_max(name)
    assert d["noise"].shape == (c["B"], c["T"], 128) and abs(d["noise"].std() - 1) < 0.2
    grads = [k for k in d.files if k.startswith("f64/")]
    assert "f64/condition" in grads and any("residual_layers.0." in k for k in grads)
    for k in grads:
        v = d[k]
        assert np.isfinite(v).all() and np.abs(v).max() > 0, k
        assert 0 < float(d["err32/" + k[4:]]) < 1e-3, k


def test_the_draw_order_is_the_references():
    """DG.draws under a seed gives the t and noise the reference's seeded forward used (the generator checked that
    replaying them reproduces that forward bit for bit): torch.randint(0, t_max, (B,)), then randn_like of the
    transposed [B, 1, M, T] view, token-major in memory"""
    for name, c in GD.CASES.items():
        if "t" in c:
            continue
        d = np.load(GD.path(name))
        torch.manual_seed(GD._seed(name))
        t, noise = DG.draws(c["B"], c["T"], GD.t_max(name))
        assert np.array_equal(t.numpy(), d["t"]) and np.array_equal(noise.contiguous().numpy(), d["noise"]), name
        assert noise.is_contiguous()                               # [B, T, M] in memory order
        torch.manual_seed(GD._seed(name))
        t2 = torch.randint(0, GD.t_max(name), (c["B"],)).long()
        x = torch.zeros(c["B"], c["T"], 128).transpose(1, 2)[:, None, :, :]
        assert torch.equal(t2, t) and torch.equal(torch.randn_like(x)[:, 0].transpose(1, 2), noise)
