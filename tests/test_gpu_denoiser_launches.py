"""Kernel launches of the two denoisers and their owners at one small shape, in each GEMM precision.

``ops.launches()`` counts the package's own kernels (the stages between the GEMMs, the TF32 splits, the column sums),
not the library GEMMs.  The training forward is the inference forward plus saved activations: same kernels, same bits
(test_gpu_reflow_backward.py, test_gpu_diffusion_backward.py).  These counts pin what runs on each path -- WaveNet and
NaiveV2Diff forward under no_grad and under grad with its backward, GaussianDiffusion's and RectifiedFlow's loss with
its backward, one DPM-Solver and one RK4 sampling call -- so a change to the shared host side that adds, drops or
reorders a launch shows up here.  Each call runs once uncounted first, so the packed weights are cached."""
import contextlib

import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import ops

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
M, MC, B, T = 32, 16, 2, 12

# per GEMM precision, the launches of each call below (3xtf32 adds the TF32 splits of the operands no kernel writes);
# the counts of the two separate host sides that the shared one (denoiser.py) replaced
_FP32 = {"wavenet_forward": 9, "wavenet_forward_backward": 30, "naive_forward": 6, "naive_forward_backward": 23,
         "diffusion_wavenet_loss_backward": 32, "diffusion_naive_loss_backward": 25, "reflow_loss_backward": 25,
         "dpm_solver_sample": 20, "rk4_sample": 50}
EXPECTED = {
    "3xtf32": {"wavenet_forward": 13, "wavenet_forward_backward": 41, "naive_forward": 12, "naive_forward_backward": 38,
               "diffusion_wavenet_loss_backward": 42, "diffusion_naive_loss_backward": 39, "reflow_loss_backward": 39,
               "dpm_solver_sample": 24, "rk4_sample": 70},
    "fp32": _FP32,
    "tf32": _FP32,
}


@contextlib.contextmanager
def precision(mode):
    prev = [(cls, cls.gemm_precision) for cls in (pkg.WaveNet, pkg.NaiveV2Diff)]
    prev_sw = pkg.WaveNet.diffusion_backward, pkg.NaiveV2Diff.reflow_backward
    for cls, _ in prev:
        cls.gemm_precision = mode
    pkg.WaveNet.diffusion_backward = pkg.NaiveV2Diff.reflow_backward = True
    try:
        yield
    finally:
        for cls, p in prev:
            cls.gemm_precision = p
        pkg.WaveNet.diffusion_backward, pkg.NaiveV2Diff.reflow_backward = prev_sw


def calls():
    """{name: a function that runs one call}: the small WaveNet and NaiveV2Diff, with every weight non-zero"""
    torch.manual_seed(0)
    nets = {"wavenet": pkg.WaveNet(M, 3, 64, MC),
            "naive": pkg.NaiveV2Diff(mel_channels=M, dim=64, num_layers=2, condition_dim=MC, use_mlp=False)}
    with torch.no_grad():
        for net in nets.values():
            for p in net.parameters():
                p.normal_(0.0, 0.1)
    nets = {k: v.to(DEV) for k, v in nets.items()}
    gd = {k: pkg.GaussianDiffusion(v, out_dims=M, timesteps=100, k_step=100).to(DEV) for k, v in nets.items()}
    flow = pkg.RectifiedFlow(nets["naive"], out_dims=M)
    spec, cond = torch.randn(B, 1, M, T, device=DEV), torch.randn(B, MC, T, device=DEV)
    cond_tm, gt = torch.randn(B, T, MC, device=DEV), torch.randn(B, T, M, device=DEV)
    x0, noise = torch.randn(B, T, M, device=DEV), torch.randn(B, 1, M, T, device=DEV)
    steps, t_int = torch.tensor([3.0, 70.0], device=DEV), torch.tensor([5, 60], device=DEV)
    t_flow = torch.tensor([0.25, 0.75], device=DEV)

    def no_grad(fn):
        def run():
            with torch.no_grad():
                fn()
        return run

    def forward_backward(net):
        def run():
            c = cond.clone().requires_grad_(True)
            out = net(spec, steps, c)
            out.backward(torch.ones_like(out))
        return run

    def loss_backward(owner, t, draw):
        def run():
            c = cond_tm.clone().requires_grad_(True)
            owner._loss(c, gt, t, draw).backward()
        return run

    out = {}
    for k, net in nets.items():
        out[k + "_forward"] = no_grad(lambda net=net: net(spec, steps, cond))
        out[k + "_forward_backward"] = forward_backward(net)
    out["diffusion_wavenet_loss_backward"] = loss_backward(gd["wavenet"], t_int, x0)
    out["diffusion_naive_loss_backward"] = loss_backward(gd["naive"], t_int, x0)
    out["reflow_loss_backward"] = loss_backward(flow, t_flow, x0)
    out["dpm_solver_sample"] = no_grad(lambda: gd["wavenet"]._sample(cond_tm, noise, gt, 20, 10, "dpm-solver"))
    out["rk4_sample"] = no_grad(lambda: flow._sample(cond_tm, noise, gt, 2, "rk4", 0.5))
    return out


def measure(mode):
    """{call: launches} at GEMM precision ``mode``"""
    got = {}
    with precision(mode):
        for name, run in calls().items():
            run()
            torch.cuda.synchronize()
            n0 = ops.launches()
            run()
            torch.cuda.synchronize()
            got[name] = ops.launches() - n0
    return got


@pytest.mark.parametrize("mode", sorted(EXPECTED))
def test_launches(mode):
    assert measure(mode) == EXPECTED[mode]
