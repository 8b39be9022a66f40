"""The mel front end's gradient oracles against the reference's own autograd gradients (tests/golden/mel_grad_*.npz,
written by tests/golden/make_golden_mel_grad.py from nvSTFT.py): oracle.mel.get_mel under autograd reproduces them bit
for bit, and the float64 restatement of the backward (tests/mel_grad_closed_form.py) matches them at the fp32 floor."""
import numpy as np
import pytest
import torch

from oracle import mel as om
from tests import mel_grad_closed_form as CF
from tests import util
from tests.golden import make_golden_mel_grad as GG

# relative RMS of the fp32 reference gradient against float64: 1.3e-6 .. 9.7e-6 on these cases (the largest on the
# clamped 172-frame row, where 1/M amplifies round-off in quiet bands)
FLOOR = 2e-5


@pytest.mark.parametrize("name", list(GG.CASES))
def test_fixture_inputs_regenerate(name):
    z = np.load(GG.path(name))
    y, hop, cot = GG.build_inputs(name)
    assert hop == int(z["hop"]) and np.array_equal(y.numpy(), z["y"]) and np.array_equal(cot.numpy(), z["cot"])


@pytest.mark.parametrize("name", list(GG.CASES))
def test_oracle_autograd_reproduces_reference_gradient(name):
    z = np.load(GG.path(name))
    y = torch.from_numpy(z["y"]).requires_grad_(True)
    mel = om.get_mel(y, hop_length=int(z["hop"]))
    assert np.array_equal(mel.detach().numpy(), z["mel"])
    (mel * torch.from_numpy(z["cot"])).sum().backward()
    assert np.array_equal(y.grad.numpy(), z["grad"])


@pytest.mark.parametrize("name", list(GG.CASES))
def test_closed_form_matches_reference_gradient(name):
    z = np.load(GG.path(name))
    ref = CF.mel_grad(z["y"], int(z["hop"]), z["cot"])
    assert ref.shape == z["grad"].shape
    e = util.rms(z["grad"] - ref) / util.rms(ref)
    assert e <= FLOOR, (name, e)
    assert np.abs(CF.log_mel(z["y"], int(z["hop"])) - z["mel"]).max() < 1e-3


def test_silent_case_exercises_the_clamp():
    z = np.load(GG.path("mel_grad_b1_f172_silence"))
    M = CF.forward(z["y"], int(z["hop"]))[2]
    assert (M < 0.5 * CF.CLIP).sum() > 1000 and (M > 2 * CF.CLIP).sum() > 10000
    # the clamp passes the gradient at equality (torch's clamp(min=) rule the kernel follows)
    x = torch.tensor([0.5e-5, 1e-5, 2e-5], requires_grad=True)
    torch.log(torch.clamp(x, min=1e-5)).sum().backward()
    assert x.grad[0] == 0 and x.grad[1] > 0 and x.grad[2] > 0


@pytest.mark.parametrize("name", ["mel_grad_b2_f12", "mel_grad_b1_short_constpad", "mel_grad_b1_f172_silence"])
def test_closed_form_equals_float64_autograd_of_the_reference_operators(name):
    z = np.load(GG.path(name))
    a = CF.mel_grad(z["y"], int(z["hop"]), z["cot"])
    b = CF.autograd64(z["y"], int(z["hop"]), z["cot"])
    assert util.rms(a - b) <= 1e-12 * util.rms(b)
