"""The diffusion oracle (tests/diffusion_oracle.py) against the reference's own sampler and denoiser outputs
(tests/golden/diffusion_*.npz, tests/golden/make_golden_diffusion.py); the package's WaveNet / GaussianDiffusion
parameter trees, buffers, step schedules and refusals -- no GPU needed."""
import json
import os

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import diffusion as pd
from tests import diffusion_oracle, util
from tests.golden import make_golden_diffusion as mk

HERE = os.path.dirname(os.path.abspath(__file__))
SAMPLER = [n for n, c in mk.CASES.items() if not c.get("net")]
NET = [n for n, c in mk.CASES.items() if c.get("net")]


def load(name):
    return {k: torch.from_numpy(v) for k, v in np.load(mk.path(name)).items()}


def run_oracle(name, dtype):
    c, d = mk.CASES[name], load(name)
    net = mk.build_oracle(c["model"]).to(dtype)
    with torch.no_grad():
        return diffusion_oracle.sample(net, d["condition"], d["noise"], d.get("gt_spec"), c["k_step"], c["speedup"],
                                       c["method"], d.get("step_noise"))


@pytest.mark.parametrize("name", SAMPLER)
def test_oracle_sampler_matches_the_reference(name):
    d = load(name)
    want = d["out32"]
    (got32, fed32), (got64, fed64) = run_oracle(name, torch.float32), run_oracle(name, torch.float64)
    assert fed32 == fed64 == d["fed"].tolist()                 # the same diffusion steps, bit for bit
    assert util.rms(got32 - want) <= 2e-6 * util.rms(want), util.rms(got32 - want) / util.rms(want)
    # float64 against the reference's fp32: the reference's own rounding through the layers and the steps
    assert util.rms(got64 - want.double()) <= 2e-5 * util.rms(want), util.rms(got64 - want.double()) / util.rms(want)


@pytest.mark.parametrize("name", NET)
def test_oracle_network_matches_the_reference(name):
    c, d = mk.CASES[name], load(name)
    net = mk.build_oracle(c["model"])
    with torch.no_grad():
        got32 = net(d["spec"], d["step"], d["cond"])
        got64 = net.double()(d["spec"].double(), d["step"].double(), d["cond"].double())
    assert got32.shape == d["out32"].shape
    assert util.rms(got32 - d["out32"]) <= 1e-6 * util.rms(d["out32"])
    assert util.rms(got64 - d["out64"]) <= 1e-12 * util.rms(d["out64"])


@pytest.mark.parametrize("name", SAMPLER)
def test_package_schedule_feeds_the_references_steps(name):
    """the package's host plan: the step values of every evaluation, bit for bit the reference's (99.0, 89.1, ... for
    DPM-Solver at k_step 100), and one evaluation per network call"""
    c, d = mk.CASES[name], load(name)
    buf = pd.GaussianDiffusion(pkg.WaveNet(128, 1, 64, 256))._host()
    t = c["k_step"] or 1000
    if c["method"] is None or c["speedup"] == 1:
        plan, _ = pd._discrete_plan(buf, t, 1, "ddpm")
    elif c["method"] in ("dpm-solver", "unipc"):
        plan, _ = pd._multistep_plan(buf["betas"][:t], t // c["speedup"], c["method"])
    else:
        plan, _ = pd._discrete_plan(buf, t, c["speedup"], c["method"])
    assert [np.float32(ev.step) for ev in plan] == [np.float32(v) for v in d["fed"].tolist()]
    assert sum(ev.emit for ev in plan) == len(plan) - 1                  # every evaluation but the last feeds the next


def test_dpm_steps_at_the_default_configuration():
    buf = pd.GaussianDiffusion(pkg.WaveNet(128, 1, 64, 256))._host()
    plan, _ = pd._multistep_plan(buf["betas"][:100], 10, "dpm-solver")
    assert [round(ev.step, 4) for ev in plan[:3]] == [99.0, 89.1, 79.2]


def test_fixture_weights_are_nonzero_and_the_outputs_depend_on_the_inputs():
    for model in mk.MODELS:
        for n, p in mk.build_oracle(model).named_parameters():
            assert (p != 0).all(), n
    d = load("diffusion_net_w64_b2_t1")["out64"]
    assert d.std() > 0.1 and (d[0] - d[1]).abs().max() > 0.1
    a, b = load("diffusion_w64_b2_t24_dpm10"), load("diffusion_w64_b2_t9_ddim10")
    for d in (a, b):                                                      # the sampler moved away from the start
        assert (d["out32"] - d["gt_spec"]).abs().max() > 0.5


def _state(module):
    return [[k, list(v.shape)] for k, v in module.state_dict().items()]


def test_package_modules_have_the_reference_state_dict_and_buffers():
    with open(os.path.join(HERE, "golden", "diffusion_state_dicts.json")) as f:
        ref = json.load(f)
    for model in mk.MODELS:
        cls, kw = mk.package_kwargs(model)
        ours = getattr(pkg, cls)(**kw)
        assert _state(ours) == ref[model]
        ours.load_state_dict(mk.build_oracle(model).state_dict(), strict=True)
    gd = pkg.GaussianDiffusion(pkg.WaveNet(**mk.package_kwargs("w64")[1]), out_dims=128)
    assert _state(gd) == ref["GaussianDiffusion_w64"]
    assert _state(pkg.GaussianDiffusion(pkg.WaveNet(128, 20, 512, 256), out_dims=128)) == ref["Unit2Wav.diff_model"]
    fast = pkg.GaussianDiffusion(pkg.NaiveV2Diff(mel_channels=128, dim=512, num_layers=6, condition_dim=128, use_mlp=False))
    assert _state(fast) == ref["Unit2WavFast.diff_model"]
    bufs = np.load(os.path.join(HERE, "golden", "diffusion_buffers.npz"))
    for name, v in gd.named_buffers():
        assert np.array_equal(v.double().numpy(), bufs[name]), name              # the same fp32 values
    assert (pkg.WaveNet(128, 1, 64, 256).output_projection.weight == 0).all()   # zero-initialised like the reference


@pytest.mark.parametrize("kw", [dict(n_chans=96), dict(n_chans=0), dict(n_layers=0)])
def test_unsupported_wavenet_options_raise_in_the_constructor(kw):
    args = dict(in_dims=128, n_layers=2, n_chans=64, n_hidden=256)
    args.update(kw)
    with pytest.raises(NotImplementedError):
        pkg.WaveNet(**args)


def test_refusals_without_a_device():
    with pytest.raises(ValueError, match="WaveNet"):
        pkg.GaussianDiffusion(mk.build_oracle("w64"))
    gd = pkg.GaussianDiffusion(pkg.WaveNet(128, 1, 64, 256))
    cond, gt = torch.zeros(1, 8, 256), torch.zeros(1, 8, 128)
    with pytest.raises(NotImplementedError, match="training"):
        gd(cond, gt_spec=gt, infer=False)
    with pytest.raises(NotImplementedError, match="training"):            # parameters require grad, grad mode on
        gd(cond, gt_spec=gt, k_step=100)
    with pytest.raises(NotImplementedError, match="training"):
        gd.denoise_fn(torch.zeros(1, 1, 128, 8), torch.zeros(1), cond.transpose(1, 2))
    with torch.no_grad(), pytest.raises(ValueError, match="CUDA"):      # no CPU fallback
        gd(cond, gt_spec=gt, k_step=100)
    with torch.no_grad(), pytest.raises(ValueError, match="CUDA"):
        gd.denoise_fn(torch.zeros(1, 1, 128, 8), torch.zeros(1), cond.transpose(1, 2))


def replay_plan(net, condition, noise, gt_spec, t, speedup, method, step_noise=None):
    """the package's host plan driven through a float64 restatement of the df_update kernel (file comment of
    csrc/diffusion.cu) with the oracle network: the per-step linear combinations against the step-by-step oracle"""
    buf = pd.GaussianDiffusion(pkg.WaveNet(128, 1, 64, 256))._host()
    if method is None or speedup == 1:
        plan, slots = pd._discrete_plan(buf, t, 1, "ddpm")
    elif method in ("dpm-solver", "unipc"):
        plan, slots = pd._multistep_plan(buf["betas"][:t], t // speedup, method)
    else:
        plan, slots = pd._discrete_plan(buf, t, speedup, method)
    B, T, _ = condition.shape
    cond = condition.double().transpose(1, 2)
    if gt_spec is None:
        x = noise.double()[:, 0].transpose(1, 2)
    else:
        nrm = (gt_spec.double() + 12) / 14 * 2 - 1
        x = float(buf["sqrt_alphas_cumprod"][t - 1]) * nrm + float(buf["sqrt_one_minus_alphas_cumprod"][t - 1]) * \
            noise.double()[:, 0].transpose(1, 2)
    point, hist, draws = x.clone(), [None] * slots, iter([] if step_noise is None else step_noise)
    for ev in plan:
        eps = net(point.transpose(1, 2)[:, None], torch.full((B,), ev.step), cond)[:, 0].transpose(1, 2)
        a_x, a_e, c_x, c_d, c1, c2, c3, cn = ev.coef
        d = a_x * x + a_e * eps
        v = c_x * x + c_d * d
        for c, s in zip((c1, c2, c3), ev.reads):
            if s is not None:
                v = v + c * hist[s]
        if ev.noise:
            v = v + cn * next(draws).double()[:, 0].transpose(1, 2)
        if ev.write is not None:
            hist[ev.write] = d
        if ev.store:
            x = v
        point = v
    return (x + 1) / 2 * 14 - 12


@pytest.mark.parametrize("name", SAMPLER)
def test_package_plan_reproduces_the_oracle_in_float64(name):
    c, d = mk.CASES[name], load(name)
    net = mk.build_oracle(c["model"]).double()
    with torch.no_grad():
        want, _ = diffusion_oracle.sample(net, d["condition"], d["noise"], d.get("gt_spec"), c["k_step"], c["speedup"],
                                          c["method"], d.get("step_noise"))
        got = replay_plan(net, d["condition"], d["noise"], d.get("gt_spec"), c["k_step"] or 1000, c["speedup"], c["method"],
                          d.get("step_noise"))
    assert util.rms(got - want) <= 1e-6 * util.rms(want), util.rms(got - want) / util.rms(want)
