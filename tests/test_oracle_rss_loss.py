"""oracle.loss (the reference's SSSLoss / RSSLoss restated on torch.stft) against the reference's own autograd goldens
(tests/golden/rss_*.npz, bit for bit), and the float64 restatement tests/rss_loss_closed_form.py against float64
autograd of the oracle."""
import numpy as np
import pytest
import torch

from oracle import loss as ol
from tests import rss_loss_closed_form as CF
from tests.golden import make_golden_rss_loss as GR


@pytest.mark.parametrize("name", list(GR.CASES))
def test_golden_inputs_regenerate(name):
    z = np.load(GR.path(name))
    x_pred, x_true, _ = GR.build_inputs(name)
    assert np.array_equal(x_pred.numpy(), z["x_pred"]) and np.array_equal(x_true.numpy(), z["x_true"])
    for k, v in GR.checksums(x_pred, x_true).items():
        assert float(z[k]) == v, k
    assert GR.draw(name).tolist() == z["n_ffts"].tolist()


@pytest.mark.parametrize("name", list(GR.CASES))
def test_oracle_reproduces_reference_bit_for_bit(name):
    z = np.load(GR.path(name))
    xp = torch.from_numpy(z["x_pred"]).requires_grad_(True)
    loss = ol.rss_loss(xp, torch.from_numpy(z["x_true"]).float(), z["n_ffts"].tolist())
    loss.backward()
    assert loss.item() == float(z["loss"])
    assert np.array_equal(xp.grad.numpy(), z["grad"])


@pytest.mark.parametrize("name", list(GR.CASES))
def test_closed_form_matches_float64_autograd(name):
    z = np.load(GR.path(name))
    x64 = torch.from_numpy(z["x_pred"]).double().requires_grad_(True)
    xt = z["x_true"].astype(np.float32)
    ref = ol.rss_loss(x64, torch.from_numpy(xt).double(), z["n_ffts"].tolist())
    ref.backward()
    loss, grad, _ = CF.loss_and_grad(z["x_pred"], xt, z["n_ffts"].tolist())
    g = x64.grad.numpy()
    assert abs(loss - ref.item()) <= 1e-12 * abs(ref.item())
    assert np.sqrt(np.mean((grad - g) ** 2)) <= 1e-11 * np.sqrt(np.mean(g ** 2))      # measured <= 1.3e-12


def test_equal_row_has_zero_gradient_in_the_reference():
    z = np.load(GR.path("rss_equal_row"))
    assert np.array_equal(z["x_pred"][1], z["x_true"][1])
    assert not np.any(z["grad"][1]) and np.any(z["grad"][0])


def test_seeded_draw_is_the_references():
    torch.manual_seed(1)
    assert ol.draw_scales(256, 2048, 4).tolist() == np.load(GR.path("rss_seeded_b2_h24"))["n_ffts"].tolist()
