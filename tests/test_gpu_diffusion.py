"""The diffusion models' WaveNet denoiser and GaussianDiffusion's five samplers on the kernels (ddsp_svc_b200/diffusion.py,
csrc/diffusion.cu) against the reference's stored outputs (tests/golden/diffusion_*.npz) and the float64 oracle
(tests/diffusion_oracle.py, run in float64 on the same GPU), at the configs' width (WaveNet(128, 20, 512, 256)).

Error metrics are relative to the truth: rms(got - truth) / rms(truth) and max|got - truth| / max|truth|.  The sampler
tests also measure the fp32 oracle run eagerly on the GPU under torch's defaults -- what the reference runs today: cuDNN
convolutions in TF32 -- and require the default "3xtf32" path to be no less accurate.  Measured errors go through
tests/report.py (B2D_PARITY_REPORT)."""
import contextlib

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import CombSubFast, FixedControls, synthetic as syn
from ddsp_svc_b200 import mel as pm
from tests import diffusion_oracle, report, util
from tests.golden import make_golden_diffusion as mk

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MODES = ("3xtf32", "fp32", "tf32")
# relative RMS / relative max bounds per GEMM mode: 2.5 to 3 times the largest error measured on an H100 80GB HBM3 at a
# 700 W power limit (DESIGN.md section 4.15).  WaveNet(128, 20, 512, 256) at 1 x 861 and 16 x 172: 3.6e-6 / 3.7e-6,
# 6.7e-7 / 9.1e-7, 7.2e-4 / 8.4e-4.  Samplers (the five on WaveNet, NaiveV2Diff with B = 3, the CombSubFast chain):
# 3.5e-6 / 5.7e-6, 2.9e-7 / 8.0e-7, 1.95e-4 / 2.56e-4; the eager fp32 reference: 1.0e-4 to 1.95e-4 / 1.4e-4 to 2.6e-4.
NET_BOUND = {"3xtf32": (1e-5, 1e-5), "fp32": (2e-6, 2.5e-6), "tf32": (2e-3, 2.5e-3)}
SAMPLER_BOUND = {"3xtf32": (1e-5, 1.5e-5), "fp32": (8e-7, 2e-6), "tf32": (5e-4, 7e-4)}
SAMPLERS = [("dpm-solver", 10), ("unipc", 10), ("pndm", 10), ("ddim", 10), (None, 1)]


def errors(got, truth):
    got, truth = got.double().cpu(), truth.double().cpu()
    return util.rms(got - truth) / util.rms(truth), float((got - truth).abs().max() / truth.abs().max())


@contextlib.contextmanager
def precision(mode):
    prev = pkg.WaveNet.gemm_precision, pkg.NaiveV2Diff.gemm_precision
    pkg.WaveNet.gemm_precision = pkg.NaiveV2Diff.gemm_precision = mode
    try:
        yield
    finally:
        pkg.WaveNet.gemm_precision, pkg.NaiveV2Diff.gemm_precision = prev


def package_model(model):
    cls, kw = mk.package_kwargs(model)
    net = getattr(pkg, cls)(**kw)
    net.load_state_dict(mk.build_oracle(model).state_dict(), strict=True)
    return pkg.GaussianDiffusion(net.to(DEV).eval(), out_dims=128).to(DEV)


_oracles = {}


def oracle(model, dtype=torch.float64):
    key = (model, dtype)
    if key not in _oracles:
        _oracles[key] = mk.build_oracle(model).to(DEV, dtype).eval()
    return _oracles[key]


def mel_inputs(B, T, seed, Mc=256, M=128):
    """a log-mel-like condition [B, T, Mc] and gt_spec [B, T, M] (a ramp over the bins plus noise)"""
    g = torch.Generator().manual_seed(seed)
    ramp = lambda n: torch.linspace(-8.0, 0.5, n)[None, None, :]
    return ((ramp(Mc) + 1.5 * torch.randn(B, T, Mc, generator=g)).to(DEV),
            (ramp(M) + 1.5 * torch.randn(B, T, M, generator=g)).to(DEV))


# ---- the reference's outputs replayed ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n, c in mk.CASES.items() if not c.get("net")])
def test_fixtures_replayed_through_the_sampler(name):
    c = mk.CASES[name]
    d = {k: torch.from_numpy(v) for k, v in np.load(mk.path(name)).items()}
    gd = package_model(c["model"])
    gt = d["gt_spec"].to(DEV) if "gt_spec" in d else None
    with torch.no_grad():
        got = gd._sample(d["condition"].to(DEV), d["noise"].to(DEV), gt, c["k_step"] or gd.k_step, c["speedup"],
                         c["method"], d.get("step_noise"))
        truth, _ = diffusion_oracle.sample(mk.build_oracle(c["model"]).double(), d["condition"], d["noise"], d.get("gt_spec"),
                                           c["k_step"], c["speedup"], c["method"], d.get("step_noise"))
    want = d["out32"]
    rel, mx = errors(got, want)
    ref_rel, ref_mx = errors(want, truth)                  # the reference's own fp32 error
    report.record("diffusion/fixture/" + name, rel_rms=rel, rel_max=mx, ref32_rel_rms=ref_rel, ref32_rel_max=ref_mx,
                  rel_rms_vs_f64=errors(got, truth)[0])
    assert got.shape == want.shape
    # measured up to 7.6e-7 / 1.3e-6 (the reference's own fp32 error on these small cases: up to 5.5e-7 / 7.1e-7)
    assert rel <= max(3.5e-6, 3 * ref_rel) and mx <= max(3.5e-6, 3 * ref_mx), (rel, mx, ref_rel, ref_mx)


@pytest.mark.parametrize("name", [n for n, c in mk.CASES.items() if c.get("net")])
def test_fixtures_replayed_through_the_network(name):
    c = mk.CASES[name]
    d = {k: torch.from_numpy(v) for k, v in np.load(mk.path(name)).items()}
    with torch.no_grad():
        got = package_model(c["model"]).denoise_fn(d["spec"].to(DEV), d["step"].to(DEV), d["cond"].to(DEV))
    rel, mx = errors(got, d["out64"])
    report.record("diffusion/fixture/" + name, rel_rms=rel, rel_max=mx)
    assert got.shape == d["out64"].shape and rel <= NET_BOUND["3xtf32"][0] and mx <= NET_BOUND["3xtf32"][1], (rel, mx)


# ---- the standalone WaveNet at the configs' width ----------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,T", [(1, 861), (16, 172)])
def test_wavenet_against_float64(mode, B, T):
    g = torch.Generator().manual_seed(B * 1000 + T)
    spec = torch.randn(B, 1, 128, T, generator=g).to(DEV)
    cond, _ = mel_inputs(B, T, B + T)
    cond = cond.transpose(1, 2).contiguous()
    steps = (100 * torch.rand(B, generator=g)).to(DEV)
    with torch.no_grad(), precision(mode):
        got = package_model("w512").denoise_fn(spec, steps, cond)
        truth = oracle("w512")(spec.double(), steps, cond.double())
    rel, mx = errors(got, truth)
    report.record("diffusion/wavenet/%s/%dx%d" % (mode, B, T), rel_rms=rel, rel_max=mx)
    assert got.shape == spec.shape
    assert rel <= NET_BOUND[mode][0] and mx <= NET_BOUND[mode][1], (rel, mx)


# ---- every sampler end to end -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method,speedup", SAMPLERS)
def test_sampler_against_float64_and_the_eager_reference(method, speedup):
    B, T = 1, 300
    cond, gt = mel_inputs(B, T, 77)
    noise = torch.randn(B, 1, 128, T, generator=torch.Generator().manual_seed(78)).to(DEV)
    steps = torch.randn(100, B, 1, 128, T, generator=torch.Generator().manual_seed(79)).to(DEV) if speedup == 1 else None
    with torch.no_grad():
        truth, _ = diffusion_oracle.sample(oracle("w512"), cond, noise, gt, 100, speedup, method, steps)
        eager, _ = diffusion_oracle.sample(oracle("w512", torch.float32), cond, noise, gt, 100, speedup, method, steps)
    e_rel, e_max = errors(eager, truth)
    res = {}
    for mode in MODES:
        with torch.no_grad(), precision(mode):
            got = package_model("w512")._sample(cond, noise, gt, 100, speedup, method, steps)
        res[mode] = errors(got, truth)
    report.record("diffusion/sampler/%s" % method, eager_rel_rms=e_rel, eager_rel_max=e_max,
                  **{"%s_rel_rms" % m: v[0] for m, v in res.items()}, **{"%s_rel_max" % m: v[1] for m, v in res.items()})
    for mode, (rel, mx) in res.items():
        assert rel <= SAMPLER_BOUND[mode][0] and mx <= SAMPLER_BOUND[mode][1], (mode, rel, mx)
    assert res["3xtf32"][0] <= e_rel and res["3xtf32"][1] <= e_max, (res["3xtf32"], (e_rel, e_max))


@pytest.mark.parametrize("method", ["dpm-solver", "pndm"])
def test_samplers_with_several_utterances_and_naive_v2_diff(method):
    """B = 3 with different lengths of content (PNDM included: the reference's branch raises for B > 1), and the
    diffusion-fast.yaml denoiser NaiveV2Diff(dim 512, 6 layers)"""
    B, T = 3, 40
    cond, gt = mel_inputs(B, T, 11, Mc=128)
    noise = torch.randn(B, 1, 128, T, generator=torch.Generator().manual_seed(12)).to(DEV)
    net = pkg.NaiveV2Diff(mel_channels=128, dim=512, num_layers=6, condition_dim=128, use_mlp=False)
    from tests import reflow_oracle
    ref = reflow_oracle.seeded_weights(reflow_oracle.VelocityNet(128, 512, 128, 6), 44)
    net.load_state_dict(ref.state_dict(), strict=True)
    with torch.no_grad():
        got = pkg.GaussianDiffusion(net.to(DEV)).to(DEV)._sample(cond, noise, gt, 100, 10, method)
        truth, _ = diffusion_oracle.sample(ref.to(DEV, torch.float64), cond, noise, gt, 100, 10, method)
        one = pkg.GaussianDiffusion(net).to(DEV)._sample(cond[1:2], noise[1:2], gt[1:2], 100, 10, method)
    rel, mx = errors(got, truth)
    report.record("diffusion/naive/%s" % method, rel_rms=rel, rel_max=mx)
    assert rel <= SAMPLER_BOUND["3xtf32"][0] and mx <= SAMPLER_BOUND["3xtf32"][1], (rel, mx)
    assert errors(one, got[1:2])[0] <= SAMPLER_BOUND["3xtf32"][0]                                # utterances do not see each other


def test_short_utterances_do_not_read_across_their_edges():
    """B = 3 with T = 1 and T = 2: each utterance alone gives its batched result"""
    gd = package_model("w512")
    for T in (1, 2):
        g = torch.Generator().manual_seed(T)
        spec, cond = torch.randn(3, 1, 128, T, generator=g).to(DEV), torch.randn(3, 256, T, generator=g).to(DEV)
        steps = torch.tensor([5.0, 50.0, 95.0], device=DEV)
        with torch.no_grad():
            both = gd.denoise_fn(spec, steps, cond)
            truth = oracle("w512")(spec.double(), steps, cond.double())
            for b in range(3):
                alone = gd.denoise_fn(spec[b:b + 1], steps[b:b + 1], cond[b:b + 1])
                assert errors(alone, both[b:b + 1])[0] <= NET_BOUND["3xtf32"][0]
        assert errors(both, truth)[0] <= NET_BOUND["3xtf32"][0]


def test_seeded_draws_match_the_oracles_order_and_runs_are_bit_identical():
    B, T = 2, 64
    cond, gt = mel_inputs(B, T, 9)
    gd = package_model("w512")
    with torch.no_grad():
        for method, speedup in (("dpm-solver", 10), (None, 1)):
            torch.manual_seed(1234)
            a = gd(cond, gt_spec=gt, infer_speedup=speedup, method=method, k_step=20)
            torch.manual_seed(1234)
            b = gd(cond, gt_spec=gt, infer_speedup=speedup, method=method, k_step=20, use_tqdm=False)
            # the reference's draws: randn_like of the transposed normalised gt_spec, then one randn per DDPM step
            torch.manual_seed(1234)
            noise = torch.randn_like(gd.norm_spec(gt).transpose(1, 2)[:, None])
            steps = [torch.randn((B, 1, 128, T), device=DEV) for _ in range(20)] if method is None else None
            truth, _ = diffusion_oracle.sample(oracle("w512"), cond, noise, gt, 20, speedup, method, steps)
            assert torch.equal(a, b)
            rel, mx = errors(a, truth)
            report.record("diffusion/seeded/%s" % method, rel_rms=rel, rel_max=mx)
            assert rel <= SAMPLER_BOUND["3xtf32"][0], (method, rel)
        torch.manual_seed(7)                                                 # the full-noise start: torch.randn
        c = gd(cond, gt_spec=None, infer_speedup=500, method="dpm-solver")
        torch.manual_seed(7)
        noise = torch.randn((B, 1, 128, T), device=DEV)
        truth, _ = diffusion_oracle.sample(oracle("w512"), cond, noise, None, None, 500, "dpm-solver")
    assert errors(c, truth)[0] <= SAMPLER_BOUND["3xtf32"][0]


def test_refusals_on_the_device():
    gd = package_model("w64")
    cond, gt = mel_inputs(1, 16, 3)
    with pytest.raises(NotImplementedError, match="training"):
        gd(cond, gt_spec=gt, infer=False)
    with pytest.raises(NotImplementedError, match="training"):             # grad mode on, parameters require grad
        gd(cond, gt_spec=gt, k_step=100)
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="heun"):
            gd(cond, gt_spec=gt, k_step=100, method="heun")
        for method in ("dpm-solver", "unipc"):                              # fewer steps than the order
            with pytest.raises(ValueError, match="at least 2 steps"):
                gd(cond, gt_spec=gt, k_step=100, method=method, infer_speedup=51)
    gd.requires_grad_(False)
    with pytest.raises(NotImplementedError, match="training"):             # an input that requires grad
        gd(cond.clone().requires_grad_(True), gt_spec=gt, k_step=100)
    gd(cond, gt_spec=gt, k_step=20, method="ddim")                         # nothing requires grad: runs


def test_ddsp_to_diffusion_chain_against_the_oracle():
    """CombSubFast -> get_mel -> GaussianDiffusion(WaveNet) with dpm-solver from k_step 100 (Unit2Wav.forward's inference
    path) from package parts, against oracle.torch_port + oracle.mel + the float64 sampler on the same controls and
    noise; WaveNet's condition here is a fixed random projection of the mel to its 256 hidden channels."""
    from oracle import mel as om
    from oracle import torch_port as tp
    SR, P = 44100, 512
    SM = syn.combsubfast_split_map(P)
    B, nF = 2, 120
    f0 = syn.make_f0(B, nF, SR, P, seed=51)
    dense, ctrls = syn.make_ctrl(B, nF, SM, seed=52)
    noise = syn.uniform_noise(B, nF * P, 53)
    proj = torch.randn(128, 256, generator=torch.Generator().manual_seed(55)).to(DEV) / 128 ** 0.5
    with torch.no_grad():
        model = CombSubFast(SR, P, unit2ctrl=FixedControls(syn.split_views(dense.to(DEV), SM), None)).to(DEV)
        signal, _, _ = model(None, f0.to(DEV), None, noise=noise.to(DEV))
        ddsp_mel = pm.STFT(SR, 128, 2048, 2048, P, 40, 16000).get_mel(signal).transpose(1, 2).contiguous()
        T = ddsp_mel.shape[1]
        x_noise = torch.randn(B, 1, 128, T, generator=torch.Generator().manual_seed(54)).to(DEV)
        got = package_model("w512")._sample((ddsp_mel @ proj).contiguous(), x_noise, ddsp_mel, 100, 10, "dpm-solver")
        ref_sig = tp.combsubfast_forward(f0, ctrls, SR, P, noise=noise)["signal"]
        ref_mel = om.get_mel(ref_sig).transpose(1, 2).to(DEV)
        truth, _ = diffusion_oracle.sample(oracle("w512"), ref_mel.double() @ proj.double(), x_noise, ref_mel, 100, 10,
                                           "dpm-solver")
    mel_rel = errors(ddsp_mel, ref_mel)[0]
    rel, mx = errors(got, truth)
    report.record("diffusion/chain", mel_rel_rms=mel_rel, rel_rms=rel, rel_max=mx)
    assert rel <= SAMPLER_BOUND["3xtf32"][0] and mx <= SAMPLER_BOUND["3xtf32"][1], (rel, mx, mel_rel)
