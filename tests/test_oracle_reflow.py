"""The reflow oracle (tests/reflow_oracle.py) against the reference's own velocity network and sampler outputs
(tests/golden/reflow_*.npz, tests/golden/make_golden_reflow.py), and the package's NaiveV2Diff / RectifiedFlow modules'
parameter trees and refusals -- no GPU needed."""
import json
import os

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from tests import reflow_oracle, util
from tests.golden import make_golden_reflow as mk

HERE = os.path.dirname(os.path.abspath(__file__))
SAMPLER = [n for n, c in mk.CASES.items() if not c.get("velocity")]
VELOCITY = [n for n, c in mk.CASES.items() if c.get("velocity")]


def load(name):
    return {k: str(v) if v.dtype.kind == "U" else torch.from_numpy(v) for k, v in np.load(mk.path(name)).items()}


def run_oracle(name, dtype):
    c, d = mk.CASES[name], load(name)
    net = mk.build_oracle(c["model"]).to(dtype)
    with torch.no_grad():
        return reflow_oracle.sample(net, d["condition"], d["noise"], d.get("gt_spec"), c["steps"], c["method"], c["t_start"])


@pytest.mark.parametrize("name", [n for n in SAMPLER if mk.CASES[n]["steps"] > 0])
def test_oracle_sampler_matches_the_reference(name):
    d = load(name)
    want = d["out32"]
    got32, got64 = run_oracle(name, torch.float32), run_oracle(name, torch.float64)
    assert util.rms(got32 - want) <= 2e-6 * util.rms(want), util.rms(got32 - want) / util.rms(want)
    # float64 against the reference's fp32: the reference's own rounding through the layer stack and the steps
    assert util.rms(got64 - want.double()) <= 5e-5 * util.rms(want)


def test_zero_steps_divide_by_zero_like_the_reference():
    name = "reflow_w128_b1_t9_euler0_t07"
    assert load(name)["raises"] == "ZeroDivisionError"
    with pytest.raises(ZeroDivisionError):
        run_oracle(name, torch.float64)


@pytest.mark.parametrize("name", VELOCITY)
def test_oracle_velocity_matches_the_reference(name):
    c, d = mk.CASES[name], load(name)
    net = mk.build_oracle(c["model"])
    with torch.no_grad():
        got32 = net(d["spec"], d["step"], d["cond"])
        got64 = net.double()(d["spec"].double(), d["step"].double(), d["cond"].double())
    assert got32.shape == d["out32"].shape
    assert util.rms(got32 - d["out32"]) <= 1e-6 * util.rms(d["out32"])
    assert util.rms(got64 - d["out64"]) <= 1e-12 * util.rms(d["out64"])


def test_fixture_weights_are_nonzero_and_the_velocity_depends_on_every_input():
    for model in mk.MODELS:
        for n, p in mk.build_oracle(model).named_parameters():
            assert (p != 0).all(), n
    d = load("reflow_vel_w128_b2_t33")
    out = d["out64"]
    assert out.std() > 0.1 and (out[0] - out[1]).abs().max() > 0.1           # different steps, inputs per utterance


def _state(module):
    return [[k, list(v.shape)] for k, v in module.state_dict().items()]


def test_package_modules_have_the_reference_state_dict():
    with open(os.path.join(HERE, "golden", "reflow_state_dicts.json")) as f:
        ref = json.load(f)
    for model in mk.MODELS:
        ours = pkg.NaiveV2Diff(use_mlp=False, **mk.model_kwargs(model))
        assert _state(ours) == ref[model]
        assert _state(mk.build_oracle(model)) == ref[model]
        ours.load_state_dict(mk.build_oracle(model).state_dict(), strict=True)
    flow = pkg.RectifiedFlow(pkg.NaiveV2Diff(use_mlp=False, **mk.model_kwargs("w512")))
    assert _state(flow) == ref["RectifiedFlow_w512"]
    assert all(k.startswith("velocity_fn.") for k, _ in ref["RectifiedFlow_w512"])
    # the reference zero-initialises the output projection; so does the package
    assert (pkg.NaiveV2Diff(use_mlp=False, dim=128, num_layers=1).output_projection.weight == 0).all()


@pytest.mark.parametrize("kw", [dict(), dict(use_mlp=True), dict(conv_only=False), dict(wavenet_like=True),
                                dict(use_norm=True), dict(conv_model_type="mode2"), dict(kernel_size=15),
                                dict(expansion_factor=4), dict(dim=96), dict(conv_dropout=0.1)])
def test_unsupported_options_raise_in_the_constructor(kw):
    args = dict(use_mlp=False, dim=128, num_layers=1)
    args.update(kw)
    if not kw:
        args.pop("use_mlp")                                   # the reference's default is use_mlp=True
    with pytest.raises(NotImplementedError):
        pkg.NaiveV2Diff(**args)


def test_sampler_refusals_without_a_device():
    net = pkg.NaiveV2Diff(use_mlp=False, dim=128, num_layers=1)
    with pytest.raises(ValueError, match="NaiveV2Diff"):
        pkg.RectifiedFlow(mk.build_oracle("w128"))
    flow = pkg.RectifiedFlow(net)
    cond = torch.zeros(1, 8, 128)
    with pytest.raises(NotImplementedError, match="training"):
        flow(cond, gt_spec=cond, infer=False)
    with pytest.raises(NotImplementedError, match="training"):            # parameters require grad, grad mode on
        flow(cond, infer=True)
    with pytest.raises(NotImplementedError, match="training"):
        net(torch.zeros(1, 128, 8), torch.zeros(1), cond.transpose(1, 2))
    with torch.no_grad(), pytest.raises(ValueError, match="CUDA"):      # no CPU fallback
        flow(cond, infer=True)
    with torch.no_grad(), pytest.raises(ValueError, match="CUDA"):
        net(torch.zeros(1, 128, 8), torch.zeros(1), cond.transpose(1, 2))
