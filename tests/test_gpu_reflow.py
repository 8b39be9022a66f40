"""The reflow model's velocity network and rectified-flow sampler on the kernels (ddsp_svc_b200/reflow.py,
csrc/reflow.cu) against the reference's stored outputs (tests/golden/reflow_*.npz) and the float64 oracle
(tests/reflow_oracle.py, run in float64 on the same GPU), at configs/reflow.yaml's width (512 channels, 6 layers).

Error metrics are relative to the truth: rms(got - truth) / rms(truth) and max|got - truth| / max|truth|.  The sampler's
tests also measure the fp32 oracle run eagerly on the GPU under torch's defaults -- what the reference runs today:
cuDNN convolutions in TF32 -- and require the default "3xtf32" path to be no less accurate.  Measured errors go through
tests/report.py (B2D_PARITY_REPORT)."""
import contextlib

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import CombSubSuperFast, FixedControls, synthetic as syn
from ddsp_svc_b200 import mel as pm
from tests import reflow_oracle, report, util
from tests.golden import make_golden_reflow as mk

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MODES = ("3xtf32", "fp32", "tf32")
# relative RMS / relative max bounds per GEMM mode: 2.5 to 3 times the largest error measured on an H100 80GB HBM3 at a
# 700 W power limit (velocity 8.7e-6 / 9.0e-6, 1.4e-6 / 1.6e-6, 1.07e-3 / 1.17e-3; sampler 1.1e-5 / 1.04e-5 (RK4 without
# gt_spec), 5.2e-7 / 5.7e-7, 7.9e-4 / 7.9e-4; DESIGN.md section 4.14)
VELOCITY_BOUND = {"3xtf32": (2.5e-5, 2.5e-5), "fp32": (4e-6, 5e-6), "tf32": (3e-3, 3e-3)}
SAMPLER_BOUND = {"3xtf32": (2.5e-5, 2.5e-5), "fp32": (1.5e-6, 1.5e-6), "tf32": (2.5e-3, 2.5e-3)}


def errors(got, truth):
    got, truth = got.double().cpu(), truth.double().cpu()
    return util.rms(got - truth) / util.rms(truth), float((got - truth).abs().max() / truth.abs().max())


@contextlib.contextmanager
def precision(mode):
    prev = pkg.NaiveV2Diff.gemm_precision
    pkg.NaiveV2Diff.gemm_precision = mode
    try:
        yield
    finally:
        pkg.NaiveV2Diff.gemm_precision = prev


def package_model(model):
    net = pkg.NaiveV2Diff(use_mlp=False, **mk.model_kwargs(model))
    net.load_state_dict(mk.build_oracle(model).state_dict(), strict=True)
    return net.to(DEV).eval()


_oracles = {}


def oracle(model, dtype=torch.float64):
    key = (model, dtype)
    if key not in _oracles:
        _oracles[key] = mk.build_oracle(model).to(DEV, dtype).eval()
    return _oracles[key]


def mel_inputs(B, T, seed, M=128):
    """a log-mel-like condition and gt_spec [B, T, M] (a ramp over the bins plus noise)"""
    g = torch.Generator().manual_seed(seed)
    ramp = torch.linspace(-8.0, 0.5, M)[None, None, :]
    return ((ramp + 1.5 * torch.randn(B, T, M, generator=g)).to(DEV),
            (ramp + 1.5 * torch.randn(B, T, M, generator=g)).to(DEV))


# ---- the reference's outputs replayed ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n, c in mk.CASES.items() if not c.get("velocity")])
def test_fixtures_replayed_through_the_sampler(name):
    c = mk.CASES[name]
    d = {k: v for k, v in np.load(mk.path(name)).items()}
    flow = pkg.RectifiedFlow(package_model(c["model"])).to(DEV)
    cond = torch.from_numpy(d["condition"]).to(DEV)
    gt = torch.from_numpy(d["gt_spec"]).to(DEV) if "gt_spec" in d else None
    with torch.no_grad():
        if c["steps"] == 0:
            with pytest.raises(ZeroDivisionError):
                flow(cond, gt_spec=gt, infer_step=0, method=c["method"], t_start=c["t_start"])
            return
        got = flow._sample(cond, torch.from_numpy(d["noise"]).to(DEV), gt, c["steps"], c["method"], c["t_start"])
        truth = reflow_oracle.sample(mk.build_oracle(c["model"]).double(), torch.from_numpy(d["condition"]),
                                     torch.from_numpy(d["noise"]), torch.from_numpy(d["gt_spec"]) if gt is not None else None,
                                     c["steps"], c["method"], c["t_start"])
    want = torch.from_numpy(d["out32"])
    rel, mx = errors(got, want)
    ref_rel, ref_mx = errors(want, truth)                  # the reference's own fp32 error
    report.record("reflow/fixture/" + name, rel_rms=rel, rel_max=mx, ref32_rel_rms=ref_rel, ref32_rel_max=ref_mx,
                  rel_rms_vs_f64=errors(got, truth)[0])
    assert got.shape == want.shape
    # measured up to 3.2e-6 / 3.9e-6 (the 3xTF32 products; the reference's own fp32 error on these small cases is 7e-7)
    assert rel <= max(1e-5, 3 * ref_rel) and mx <= max(1e-5, 3 * ref_mx), (rel, mx, ref_rel, ref_mx)


@pytest.mark.parametrize("name", [n for n, c in mk.CASES.items() if c.get("velocity")])
def test_fixtures_replayed_through_the_velocity_network(name):
    c = mk.CASES[name]
    d = {k: torch.from_numpy(v) for k, v in np.load(mk.path(name)).items()}
    with torch.no_grad():
        got = package_model(c["model"])(d["spec"].to(DEV), d["step"].to(DEV), d["cond"].to(DEV))
    rel, mx = errors(got, d["out64"])
    report.record("reflow/fixture/" + name, rel_rms=rel, rel_max=mx)
    assert got.shape == d["out64"].shape and rel <= 1e-5 and mx <= 1e-5, (rel, mx)                 # measured 3.9e-6 / 4.3e-6


# ---- the standalone velocity network at reflow.yaml's width -----------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,T,four", [(1, 861, True), (48, 172, False)])
def test_velocity_network_against_float64(mode, B, T, four):
    g = torch.Generator().manual_seed(B * 1000 + T)
    spec = torch.randn(B, 128, T, generator=g).to(DEV)
    cond, _ = mel_inputs(B, T, B + T)
    cond = cond.transpose(1, 2).contiguous()
    steps = (1000 * torch.rand(B, generator=g)).to(DEV)                    # one diffusion step per utterance
    x = spec[:, None] if four else spec
    with torch.no_grad(), precision(mode):
        got = package_model("w512")(x, steps, cond)
        truth = oracle("w512")(x.double(), steps, cond.double())
    assert got.shape == x.shape
    rel, mx = errors(got, truth)
    report.record("reflow/velocity/%s/%dx%d" % (mode, B, T), rel_rms=rel, rel_max=mx)
    assert rel <= VELOCITY_BOUND[mode][0] and mx <= VELOCITY_BOUND[mode][1], (rel, mx)


# ---- the full sampler ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method,steps", [("euler", 20), ("rk4", 5)])
def test_sampler_against_float64_and_the_eager_reference(method, steps):
    B, T = 1, 861
    cond, gt = mel_inputs(B, T, 77)
    noise = torch.randn(B, 1, 128, T, generator=torch.Generator().manual_seed(78)).to(DEV)
    with torch.no_grad():
        truth = reflow_oracle.sample(oracle("w512"), cond, noise, gt, steps, method, 0.7)
        eager = reflow_oracle.sample(oracle("w512", torch.float32), cond, noise, gt, steps, method, 0.7)   # torch defaults
    e_rel, e_max = errors(eager, truth)
    res = {}
    for mode in MODES:
        with torch.no_grad(), precision(mode):
            flow = pkg.RectifiedFlow(package_model("w512"))
            got = flow._sample(cond, noise, gt, steps, method, 0.7)
        res[mode] = errors(got, truth)
    report.record("reflow/sampler/%s%d" % (method, steps), eager_rel_rms=e_rel, eager_rel_max=e_max,
                  **{"%s_rel_rms" % m: v[0] for m, v in res.items()}, **{"%s_rel_max" % m: v[1] for m, v in res.items()})
    for mode, (rel, mx) in res.items():
        assert rel <= SAMPLER_BOUND[mode][0] and mx <= SAMPLER_BOUND[mode][1], (mode, rel, mx)
    assert res["3xtf32"][0] <= e_rel and res["3xtf32"][1] <= e_max, (res["3xtf32"], (e_rel, e_max))


def test_sampler_without_gt_spec_against_float64():
    B, T = 2, 300
    cond, _ = mel_inputs(B, T, 5)
    noise = torch.randn(B, 1, 128, T, generator=torch.Generator().manual_seed(6)).to(DEV)
    with torch.no_grad():
        got = pkg.RectifiedFlow(package_model("w512"))._sample(cond, noise, None, 4, "rk4", 0.0)
        truth = reflow_oracle.sample(oracle("w512"), cond, noise, None, 4, "rk4", 0.0)
    rel, mx = errors(got, truth)
    report.record("reflow/sampler/nogt_rk4", rel_rms=rel, rel_max=mx)
    assert rel <= SAMPLER_BOUND["3xtf32"][0] and mx <= SAMPLER_BOUND["3xtf32"][1], (rel, mx)


def test_seeded_noise_matches_the_references_draw_and_runs_are_bit_identical():
    B, T = 2, 97
    cond, gt = mel_inputs(B, T, 9)
    flow = pkg.RectifiedFlow(package_model("w512"))
    with torch.no_grad():
        torch.manual_seed(1234)
        a = flow(cond, gt_spec=gt, infer_step=3, method="euler", t_start=0.7)
        torch.manual_seed(1234)
        b = flow(cond, gt_spec=gt, infer_step=3, method="euler", t_start=0.7, use_tqdm=False)
        torch.manual_seed(1234)
        noise = torch.randn((B, 1, 128, T), device=DEV)                      # reflow/reflow.py:80's draw
        c = flow._sample(cond, noise, gt, 3, "euler", 0.7)
        truth = reflow_oracle.sample(oracle("w512"), cond, noise, gt, 3, "euler", 0.7)
        torch.manual_seed(1234)
        d = flow(cond, gt_spec=None, infer_step=2, method="rk4")
        torch.manual_seed(1234)
        e = flow._sample(cond, torch.randn((B, 1, 128, T), device=DEV), None, 2, "rk4", 0.0)
    assert torch.equal(a, b) and torch.equal(a, c) and torch.equal(d, e)
    assert errors(a, truth)[0] <= SAMPLER_BOUND["3xtf32"][0]
    with torch.no_grad():                                                    # negative t_start clamps to 0
        torch.manual_seed(5)
        f = flow(cond, gt_spec=gt, infer_step=2, t_start=-0.5)
        torch.manual_seed(5)
        g = flow(cond, gt_spec=gt, infer_step=2, t_start=0.0)
    assert torch.equal(f, g)


def test_refusals_on_the_device():
    flow = pkg.RectifiedFlow(package_model("w128"))
    cond, gt = mel_inputs(1, 16, 3)
    with pytest.raises(NotImplementedError, match="training"):
        flow(cond, gt_spec=gt, infer=False)
    with pytest.raises(NotImplementedError, match="training"):             # grad mode on, parameters require grad
        flow(cond, gt_spec=gt)
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="heun"):
            flow(cond, gt_spec=gt, method="heun")
    flow.requires_grad_(False)
    with pytest.raises(NotImplementedError, match="training"):             # an input that requires grad
        flow(cond.clone().requires_grad_(True), gt_spec=gt)
    flow(cond, gt_spec=gt, infer_step=1)                                    # no parameter or input requires grad: runs


def test_ddsp_to_sampler_chain_against_the_oracle():
    """CombSubSuperFast -> get_mel -> RectifiedFlow (Unit2Wav.forward's inference path with t_start 0.7, 20 Euler
    steps) from package parts, against oracle.torch_port + oracle.mel + the float64 sampler on the same controls and
    noise."""
    from oracle import mel as om
    from oracle import torch_port as tp
    SR, P, WIN = 44100, 512, 2048
    SM = syn.superfast_split_map(WIN)
    B, nF = 2, 120
    f0 = syn.make_f0(B, nF, SR, P, seed=51)
    dense, ctrls = syn.make_ctrl(B, nF, SM, seed=52)
    noise = syn.normal_noise((B, nF * P), 53)
    with torch.no_grad():
        model = CombSubSuperFast(SR, P, WIN, unit2ctrl=FixedControls(syn.split_views(dense.to(DEV), SM),
                                                                     torch.zeros(B, nF, 256, device=DEV))).to(DEV)
        signal, _, _ = model(None, f0.to(DEV), None, noise=noise.to(DEV))
        ddsp_mel = pm.STFT(SR, 128, 2048, 2048, P, 40, 16000).get_mel(signal).transpose(1, 2).contiguous()
        T = ddsp_mel.shape[1]
        x_noise = torch.randn(B, 1, 128, T, generator=torch.Generator().manual_seed(54)).to(DEV)
        got = pkg.RectifiedFlow(package_model("w512"))._sample(ddsp_mel, x_noise, ddsp_mel, 20, "euler", 0.7)
        ref_sig = tp.superfast_forward(f0, ctrls, SR, P, WIN, noise=noise)["signal"]
        ref_mel = om.get_mel(ref_sig).transpose(1, 2).to(DEV)
        truth = reflow_oracle.sample(oracle("w512"), ref_mel, x_noise, ref_mel, 20, "euler", 0.7)
    mel_rel = errors(ddsp_mel, ref_mel)[0]
    rel, mx = errors(got, truth)
    report.record("reflow/chain", mel_rel_rms=mel_rel, rel_rms=rel, rel_max=mx)
    assert rel <= 1.5e-5 and mx <= 1.5e-5, (rel, mx, mel_rel)                                     # measured 4.6e-6 / 5.3e-6
