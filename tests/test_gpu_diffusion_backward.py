"""The diffusion loss and the WaveNet denoiser's CUDA backward (csrc/diffusion_bwd.cu + reflow_bwd.cu's loss + library
GEMMs, ddsp_svc_b200/diffusion.py: _DiffusionLossFunction, _WaveNetFunction) on the GPU:

* the diffusion-new.yaml network (WaveNet(128, 20, 512, 256)) at its training batch (36 x 172) and at 1 x 861, and the
  diffusion-fast.yaml denoiser (NaiveV2Diff(512, 6 layers)) inside GaussianDiffusion at 48 x 172, against float64
  autograd of the oracle (tests/diffusion_grad_oracle.py) on the same GPU; the default 3xTF32 path must be closer to
  float64 than the same oracle in eager fp32 under torch's defaults (cuDNN TF32 convolutions);
* each new kernel alone through the C ABI at real shapes against float64, run twice (bit-identical);
* the training forward is the no_grad forward, determinism, the reference's draws, the switch and the refusals;
* the reference's own loss and float64 gradients replayed (tests/golden/diffusion_grad_*.npz) in the three GEMM modes;
* AdamW steps through GaussianDiffusion(infer=False): the loss falls and the packed weights are rebuilt every step;
* end to end: a diffusion-new.yaml step from package parts (CombSubFast with its own Unit2Control, pcmer_backward on,
  infer=False -> get_mel -> mse, plus the diffusion loss on the control network's hidden output -> backward through all
  of it) against the oracle chain fed the same draws, then AdamW steps.

Errors are relative RMS against float64 per tensor, recorded through tests/report.py (B2D_PARITY_REPORT)."""
import contextlib
import json

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import _lib, ops
from tests import diffusion_grad_oracle as DG
from tests import report, util
from tests.golden import make_golden_diffusion as mk
from tests.golden import make_golden_diffusion_grad as GD
from tests.golden import make_golden_reflow as mkr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MODES = ("3xtf32", "fp32", "tf32")
# Bounds are about 3 times the largest error measured on an H100 80GB HBM3 at 700 W (DESIGN.md section 4.15b).
# Worst parameter tensor (w512 at 36 x 172): fp32 3.0e-7, 3xtf32 4.4e-5 (a dilated_conv.weight), tf32 1.6e-3; NaiveV2Diff
# at 48 x 172 3.0e-5.  The condition's cotangent sums every layer's products over n_layers 2 C = 20480 columns with
# heavy cancellation at this case: fp32 1.6e-6, 3xtf32 4.3e-4 (1.5e-5 at 1 x 861), tf32 1.9e-2, and eager fp32 under
# torch's defaults 1.9e-2.  Loss: 3.0e-8 / 9.7e-7 / 2.2e-5.
NETWORK_BOUND = {"fp32": 1e-6, "3xtf32": 1.5e-4, "tf32": 5e-3}
CONDITION_BOUND = {"fp32": 5e-6, "3xtf32": 1.5e-3, "tf32": 6e-2}


def rel(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return util.rms(got - want) / max(util.rms(want), 1e-300)


@contextlib.contextmanager
def training(mode="3xtf32"):
    prev = (pkg.WaveNet.gemm_precision, pkg.WaveNet.diffusion_backward, pkg.NaiveV2Diff.gemm_precision,
            pkg.NaiveV2Diff.reflow_backward)
    pkg.WaveNet.gemm_precision, pkg.WaveNet.diffusion_backward = mode, True
    pkg.NaiveV2Diff.gemm_precision, pkg.NaiveV2Diff.reflow_backward = mode, True
    try:
        yield
    finally:
        (pkg.WaveNet.gemm_precision, pkg.WaveNet.diffusion_backward, pkg.NaiveV2Diff.gemm_precision,
         pkg.NaiveV2Diff.reflow_backward) = prev


def oracle_net(model):
    """("w64" / "w512": make_golden_diffusion's seeded WaveNets; "naive512": the diffusion-fast.yaml NaiveV2Diff(512,
    6 layers, condition 128) with make_golden_reflow's seeded weights) -> fp32 CPU oracle"""
    return mkr.build_oracle("w512") if model == "naive512" else mk.build_oracle(model)


def package_diffusion(model):
    if model == "naive512":
        net = pkg.NaiveV2Diff(use_mlp=False, **mkr.model_kwargs("w512"))
    else:
        cls, kw = mk.package_kwargs(model)
        net = getattr(pkg, cls)(**kw)
    net.load_state_dict(oracle_net(model).state_dict(), strict=True)
    return pkg.GaussianDiffusion(net.to(DEV), out_dims=128).to(DEV)


def cond_width(model):
    return 128 if model == "naive512" else 256


def mel_inputs(B, T, seed, Mc=256, M=128):
    g = torch.Generator().manual_seed(seed)
    ramp = lambda n: torch.linspace(-8.0, 0.5, n)[None, None, :]
    return ((ramp(Mc) + 1.5 * torch.randn(B, T, Mc, generator=g)).to(DEV),
            (ramp(M) + 1.5 * torch.randn(B, T, M, generator=g)).to(DEV))


def seeded_draws(B, T, seed, t_max=100):
    torch.manual_seed(seed)
    return DG.draws(B, T, t_max, device=DEV)


def package_gradients(diff, cond, gt, t, noise):
    diff.zero_grad(set_to_none=True)
    c = cond.clone().requires_grad_(True)
    loss = diff._loss(c, gt, t, noise)
    loss.backward()
    grads = {n: p.grad for n, p in diff.denoise_fn.named_parameters()}
    grads["condition"] = c.grad
    return loss.detach(), grads


def oracle_gradients(model, cond, gt, t, noise, dtype=torch.float64):
    net = oracle_net(model).to(DEV, dtype)
    c = cond.to(dtype).clone().requires_grad_(True)
    loss = DG.oracle_loss(net, c, gt, t, noise)
    loss.backward()
    grads = {n: p.grad for n, p in net.named_parameters()}
    grads["condition"] = c.grad
    return loss.detach(), grads


# ---- the reference's gradients replayed ----------------------------------------------------------------------------------
# Fixtures (w64 WaveNet, w128 NaiveV2Diff; the stored entries): each tensor within max(3 err32, floor), err32 the
# reference's own fp32 error over the same entries.
# Measured worst tensors: fp32 1.0e-5, 3xtf32 1.0e-5, tf32 1.6e-2 (the input projection: one TF32 pass rounds every
# operand to 11 bits and its cotangent goes through every layer); loss 1.2e-7 / 1.8e-6 / 1.4e-4.
FIXTURE_FLOOR = {"fp32": 3e-5, "3xtf32": 3e-5, "tf32": 5e-2}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(GD.CASES))
def test_fixture_loss_and_gradients(name, mode):
    d = np.load(GD.path(name))
    dev = lambda k: torch.from_numpy(d[k]).to(DEV)
    with training(mode):
        diff = package_diffusion(GD.CASES[name]["model"])
        loss, grads = package_gradients(diff, dev("condition"), dev("gt_spec"), dev("t"), dev("noise"))
    loss64, loss32 = float(d["loss64"]), float(d["loss32"])
    loss_err, ref_loss_err = abs(loss.item() - loss64) / loss64, abs(loss32 - loss64) / loss64
    errs, over = {}, {}
    assert {n for n, g in grads.items() if g is None} == set(json.loads(str(d["none"])))
    for n, g in GD.stored(name, grads).items():
        errs[n] = rel(g, torch.from_numpy(d["f64/" + n]))
        bound = max(3 * float(d["err32/" + n]), FIXTURE_FLOOR[mode])
        if not errs[n] <= bound:
            over[n] = (errs[n], bound)
    report.record("diffusion_backward/fixture/%s/%s" % (name, mode), loss=loss_err, ref32_loss=ref_loss_err,
                  max_grad=max(errs.values()), **errs)
    assert loss_err <= max(3 * ref_loss_err, FIXTURE_FLOOR[mode]), (loss_err, ref_loss_err)
    assert not over, over


# ---- the configurations' networks against float64 ------------------------------------------------------------------------
@pytest.mark.parametrize("model,mode,B,T", [("w512", "3xtf32", 36, 172), ("w512", "fp32", 36, 172),
                                            ("w512", "tf32", 36, 172), ("w512", "3xtf32", 1, 861),
                                            ("naive512", "3xtf32", 48, 172)])
def test_network_gradients_against_float64(model, mode, B, T):
    cond, gt = mel_inputs(B, T, B + T, Mc=cond_width(model))
    t, noise = seeded_draws(B, T, 7 + B)
    with training(mode):
        diff = package_diffusion(model)
        loss, grads = package_gradients(diff, cond, gt, t, noise)
    del diff
    loss64, want = oracle_gradients(model, cond, gt, t, noise)
    errs = {n: rel(g, want[n]) for n, g in grads.items() if want[n] is not None}
    assert all(grads[n] is None for n, w in want.items() if w is None)
    params = {n: e for n, e in errs.items() if n != "condition"}
    rec = dict(loss=rel(loss, loss64), max_grad=max(errs.values()), max_param_grad=max(params.values()), **errs)
    eager_errs = None
    if mode == "3xtf32" and T == 172:
        # eager fp32 under torch's defaults (cuDNN TF32 convolutions): what the reference trains with today
        loss32, eager = oracle_gradients(model, cond, gt, t, noise, dtype=torch.float32)
        eager_errs = {n: rel(g, want[n]) for n, g in eager.items() if want[n] is not None}
        rec.update(eager_loss=rel(loss32, loss64), eager_max_grad=max(eager_errs.values()),
                   eager_condition=eager_errs["condition"])
    report.record("diffusion_backward/%s/%s/%dx%d" % (model, mode, B, T), **rec)
    if eager_errs is not None:
        assert max(errs.values()) < max(eager_errs.values()), (max(errs.values()), max(eager_errs.values()))
    bound = NETWORK_BOUND[mode]
    assert rel(loss, loss64) <= bound
    assert max(params.values()) <= bound, {n: e for n, e in params.items() if e > bound}
    assert errs["condition"] <= CONDITION_BOUND[mode], errs["condition"]


# ---- the kernels alone -------------------------------------------------------------------------------------------------
def _twice(fn):
    a, b = fn(), fn()
    for x, y in zip(a, b):
        assert torch.isfinite(x).all() and torch.equal(x, y)
    return a


def _rand(*shape, seed, scale=1.0):
    return (scale * torch.randn(*shape, generator=torch.Generator().manual_seed(seed))).to(DEV)


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


@pytest.mark.parametrize("B,T", [(36, 172), (32, 861)])
def test_loss_input_relu_mish_and_gate_kernels(B, T):
    L, M, C, nL, st = _lib.lib(), 128, 512, 20, ops._stream()
    N, Z2 = B * T, 2 * 512 * 20
    gt, noise = _rand(B, T, M, seed=1, scale=3), _rand(B, T, M, seed=2)
    t = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(3)).to(DEV)
    tb = DG.diffusion_oracle.tables()
    sa, s1m = tb["sqrt_alphas_cumprod"].to(DEV), tb["sqrt_one_minus_alphas_cumprod"].to(DEV)
    gy, pre, bias = _rand(N, C, seed=4), _rand(N, C, seed=5, scale=2), _rand(C, seed=6)
    gm, xm = _rand(B, 4 * C, seed=7), _rand(B, 4 * C, seed=8, scale=3)
    ga, g, cond = _rand(N, C, seed=9), _rand(N, 2 * C, seed=10, scale=2), _rand(N, Z2, seed=11)
    layer = 7

    def run():
        xh, xl = _nan(B, T, M), _nan(B, T, M)
        _lib.check(L.b2d_df_loss_input(gt.data_ptr(), noise.data_ptr(), t.data_ptr(), sa.data_ptr(), s1m.data_ptr(), 1000,
                                       -12.0, 14.0, B, T, M, xh.data_ptr(), xl.data_ptr(), st), "df_loss_input")
        gx, rh, rl = _nan(N, C), _nan(N, C), _nan(N, C)
        _lib.check(L.b2d_df_relu_backward(gy.data_ptr(), pre.data_ptr(), bias.data_ptr(), N, C, gx.data_ptr(), rh.data_ptr(),
                                          rl.data_ptr(), st), "df_relu_backward")
        gmx = _nan(B, 4 * C)
        _lib.check(L.b2d_df_mish_backward(gm.data_ptr(), xm.data_ptr(), B * 4 * C, gmx.data_ptr(), 0, 0, st),
                   "df_mish_backward")
        gz, zh, zl = torch.zeros(N, Z2, device=DEV), torch.zeros(N, Z2, device=DEV), torch.zeros(N, Z2, device=DEV)
        _lib.check(L.b2d_df_gate_backward(ga.data_ptr(), g.data_ptr(), cond.data_ptr() + 4 * layer * 2 * C, Z2, N, C, layer,
                                          nL, gz.data_ptr(), zh.data_ptr(), zl.data_ptr(), st), "df_gate_backward")
        return xh, xl, gx, rh, rl, gmx, gz, zh, zl

    xh, xl, gx, rh, rl, gmx, gz, zh, zl = _twice(run)
    d = lambda v: v.double()
    x0 = (d(gt) + 12) / 14 * 2 - 1
    want_x = d(sa)[t][:, None, None] * x0 + d(s1m)[t][:, None, None] * d(noise)
    x = (d(pre) + d(bias)).requires_grad_(True)
    torch.relu(x).backward(d(gy))
    y = d(xm).requires_grad_(True)
    torch.nn.functional.mish(y).backward(d(gm))
    blk = slice(layer * 2 * C, (layer + 1) * 2 * C)
    z = (d(g) + d(cond)[:, blk]).requires_grad_(True)
    (torch.sigmoid(z[:, :C]) * torch.tanh(z[:, C:])).backward(d(ga))
    e = {"x_t": rel(d(xh) + d(xl), want_x), "relu": rel(gx, x.grad), "relu_halves": rel(d(rh) + d(rl), x.grad),
         "mish": rel(gmx, y.grad), "gate": rel(gz[:, blk], z.grad), "gate_halves": rel(d(zh[:, blk]) + d(zl[:, blk]), z.grad)}
    assert not gz[:, :blk.start].any() and not gz[:, blk.stop:].any()
    report.record("diffusion_backward/kernels/pointwise/%dx%d" % (B, T), **e)
    assert max(e.values()) <= 1e-6, e


@pytest.mark.parametrize("B,T", [(36, 172), (32, 861)])
def test_layer_backward_kernel(B, T):
    L, C, nL, st = _lib.lib(), 512, 20, ops._stream()
    N, LC, div = B * T, 512 * 20, float(np.sqrt(20.0))
    gus = [_rand(N, 3 * C, seed=20 + i) for i in (nL - 1, nL - 2)]
    gsk = _rand(N, C, seed=14)
    n = L.b2d_rf_backward_workspace_bytes(B, T, LC)
    ws = torch.zeros(n, dtype=torch.uint8, device=DEV)

    def run():
        gh, gr, hi, lo = _nan(N, C), _nan(N, 2 * C), _nan(N, 2 * C), _nan(N, 2 * C)
        _lib.check(L.b2d_df_layer_backward(0, gh.data_ptr(), gsk.data_ptr(), div, B, T, C, nL - 1, nL, gr.data_ptr(),
                                           hi.data_ptr(), lo.data_ptr(), 0, 0, st), "df_layer_backward")
        for k, i in enumerate((nL - 1, nL - 2)):
            _lib.check(L.b2d_df_layer_backward(gus[k].data_ptr(), gh.data_ptr(), gsk.data_ptr(), div, B, T, C, i, nL,
                                               gr.data_ptr(), hi.data_ptr(), lo.data_ptr(), ws.data_ptr(), n, st),
                       "df_layer_backward")
        gS = torch.zeros(B, LC, device=DEV)
        _lib.check(L.b2d_rf_step_sums(ws.data_ptr(), n, B, T, LC, gS.data_ptr(), st), "rf_step_sums")
        return gh, gr, hi, lo, gS[:, (nL - 2) * C:]

    gh, gr, hi, lo, gS = _twice(run)
    d = lambda v: v.double()
    h = torch.zeros(N, C, dtype=torch.float64, device=DEV)
    sums = []
    for gu in gus:
        u = d(gu).reshape(B, T, 3, C)
        gy = u[:, :, 1].clone()
        gy[:, :-1] += u[:, 1:, 0]
        gy[:, 1:] += u[:, :-1, 2]
        h = h / np.sqrt(2) + gy.reshape(N, C)
        sums.insert(0, gy.sum(1))
    want_r = torch.cat([h / np.sqrt(2), d(gsk) / div], dim=1)
    e = {"gh": rel(gh, h), "gr": rel(gr, want_r), "gr_halves": rel(d(hi) + d(lo), want_r),
         "step_sums": rel(gS, torch.cat(sums, dim=1))}
    report.record("diffusion_backward/kernels/layer/%dx%d" % (B, T), **e)
    assert max(e.values()) <= 1e-6, e


# ---- the training forward, determinism, draws, refusals ------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_training_forward_is_the_no_grad_forward(mode):
    B, T = 3, 70
    cond, gt = mel_inputs(B, T, 31)
    spec = torch.randn(B, 128, T, generator=torch.Generator().manual_seed(32)).to(DEV)
    steps = torch.tensor([10, 500, 999], device=DEV)
    t, noise = seeded_draws(B, T, 33, 1000)
    with training(mode):
        diff = package_diffusion("w512")
        net = diff.denoise_fn
        with torch.no_grad():
            v0 = net(spec[:, None], steps, cond.transpose(1, 2))
            l0 = diff._loss(cond, gt, t, noise)
        v1 = net(spec[:, None], steps, cond.transpose(1, 2))
        l1 = diff._loss(cond, gt, t, noise)
        c = cond.clone().requires_grad_(True)
        net.requires_grad_(False)
        v2 = net(spec, steps, c.transpose(1, 2))                  # only cond requires grad
        l2 = diff._loss(c, gt, t, noise)
    assert v1.requires_grad and l1.requires_grad and v2.requires_grad and l2.requires_grad and not v0.requires_grad
    assert torch.equal(v0, v1) and torch.equal(v0, v2) and torch.equal(l0, l1) and torch.equal(l0, l2)


@pytest.mark.parametrize("model", ["w512", "naive512"])
def test_two_backwards_and_two_runs_are_bit_identical(model):
    B, T = 4, 150
    cond, gt = mel_inputs(B, T, 41, Mc=cond_width(model))
    t, noise = seeded_draws(B, T, 42)
    with training():
        diff = package_diffusion(model)
        params = [p for n, p in diff.denoise_fn.named_parameters() if ".norm." not in n]
        c = cond.clone().requires_grad_(True)
        loss = diff._loss(c, gt, t, noise)
        a = torch.autograd.grad(loss, params + [c], retain_graph=True)
        b = torch.autograd.grad(loss, params + [c])
        c2 = cond.clone().requires_grad_(True)
        d = torch.autograd.grad(diff._loss(c2, gt, t, noise), params + [c2])
        if model == "w512":
            spec = noise.transpose(1, 2).contiguous()
            cot = torch.randn(B, 1, 128, T, generator=torch.Generator().manual_seed(43)).to(DEV)
            e = torch.autograd.grad((diff.denoise_fn(spec, t, c.transpose(1, 2)) * cot).sum(), params + [c])
            f = torch.autograd.grad((diff.denoise_fn(spec, t, c.transpose(1, 2)) * cot).sum(), params + [c])
            assert all(torch.equal(x, y) for x, y in zip(e, f))
    assert all(torch.equal(x, y) and torch.equal(x, z) for x, y, z in zip(a, b, d))


def test_wavenet_forward_under_grad_against_float64():
    """WaveNet's own forward under grad, with a random cotangent: every parameter's and cond's gradient"""
    B, T = 2, 61
    cond, _ = mel_inputs(B, T, 45)
    spec = torch.randn(B, 1, 128, T, generator=torch.Generator().manual_seed(46)).to(DEV)
    steps = torch.tensor([3.0, 871.5], device=DEV)
    cot = torch.randn(B, 1, 128, T, generator=torch.Generator().manual_seed(47)).to(DEV)
    with training():
        net = package_diffusion("w64").denoise_fn
        c = cond.transpose(1, 2).contiguous().requires_grad_(True)
        (net(spec, steps, c) * cot).sum().backward()
    ref = oracle_net("w64").to(DEV, torch.float64)
    c64 = cond.transpose(1, 2).double().contiguous().requires_grad_(True)
    (ref(spec.double(), steps, c64) * cot.double()).sum().backward()
    errs = {n: rel(p.grad, q.grad) for (n, p), (_, q) in zip(net.named_parameters(), ref.named_parameters())}
    errs["cond"] = rel(c.grad, c64.grad)
    report.record("diffusion_backward/wavenet_forward_w64", **errs)
    assert max(errs.values()) <= 1e-4, errs


def test_seeded_draws_are_the_references_expressions():
    """forward(infer=False) under a seed equals _loss fed the reference's own expressions: t = torch.randint(0, t_max,
    (B,)), then noise = torch.randn_like of the transposed [B, 1, M, T] view of norm(gt_spec) (diffusion.py:220-234,
    :205); t_max is k_step, or self.k_step when k_step is None"""
    B, T = 3, 50
    cond, gt = mel_inputs(B, T, 51)
    with training():
        diff = package_diffusion("w64")
        with torch.no_grad():
            for k_step, t_max in ((100, 100), (None, 1000)):
                torch.manual_seed(52)
                a = diff(cond, gt_spec=gt, infer=False, k_step=k_step)
                torch.manual_seed(52)
                t = torch.randint(0, t_max, (B,), device=DEV).long()
                x0 = ((gt - (-12)) / (2 - (-12)) * 2 - 1).transpose(1, 2)[:, None, :, :]
                noise = torch.randn_like(x0)
                b = diff._loss(cond, gt, t, noise[:, 0].transpose(1, 2))
                assert torch.equal(a, b)
                assert noise.stride(0) == T * 128 and noise.stride()[2:] == (1, 128)      # token-major
            torch.manual_seed(53)
            e = diff(cond, gt_spec=gt, infer=False, k_step=100)
        torch.manual_seed(52)
        f = diff(cond, gt_spec=gt, infer=False, k_step=None)          # under grad: the same value
    assert not torch.equal(a, e) and torch.equal(a, f.detach()) and f.requires_grad


def test_switch_and_refusals():
    assert pkg.WaveNet.diffusion_backward is False and pkg.NaiveV2Diff.reflow_backward is False
    diff = package_diffusion("w64")
    cond, gt = mel_inputs(2, 20, 61)
    t, noise = seeded_draws(2, 20, 62)
    with pytest.raises(NotImplementedError, match="WaveNet.diffusion_backward"):
        diff(cond, gt_spec=gt, infer=False)
    with pytest.raises(NotImplementedError, match="training"):
        diff._loss(cond, gt, t, noise)
    with pytest.raises(NotImplementedError, match="training"):
        diff.denoise_fn(noise.transpose(1, 2), t, cond.transpose(1, 2))
    diff.denoise_fn.diffusion_backward = True                       # per instance
    loss = diff(cond, gt_spec=gt, infer=False)
    assert loss.requires_grad and loss.dim() == 0
    with pytest.raises(NotImplementedError, match="not differentiable"):
        diff(cond, gt_spec=gt, k_step=100)
    with pytest.raises(NotImplementedError, match="spec"):
        diff.denoise_fn(noise.transpose(1, 2).clone().requires_grad_(True), t, cond.transpose(1, 2))
    with pytest.raises(NotImplementedError, match="data"):
        diff._loss(cond, gt.clone().requires_grad_(True), t, noise)
    with pytest.raises(ValueError, match="int64"):
        diff._loss(cond, gt, t.float(), noise)
    for k_step in (0, 1001):                                        # outside the schedule: refused on the host
        with pytest.raises(ValueError, match="k_step"):
            diff(cond, gt_spec=gt, infer=False, k_step=k_step)
    with pytest.raises(ValueError, match="gt_spec"):
        diff(cond, gt_spec=None, infer=False)
    with pytest.raises(ValueError, match="float32"):
        diff._loss(cond.half(), gt, t, noise)
    assert pkg.WaveNet.diffusion_backward is False
    with torch.no_grad():
        diff(cond, gt_spec=gt, k_step=20, method="ddim")           # the sampler still runs without grad
    naive = package_diffusion("naive512")
    cn, _ = mel_inputs(2, 20, 63, Mc=128)
    with pytest.raises(NotImplementedError, match="reflow_backward"):
        naive(cn, gt_spec=gt, infer=False)
    naive.denoise_fn.reflow_backward = True                         # NaiveV2Diff's own switch, no second one
    assert naive(cn, gt_spec=gt, infer=False).requires_grad


def test_adamw_steps_repack_the_weights():
    """optimizer.step() changes every parameter in place: the packed weights are rebuilt (keyed on _version) and the
    loss falls"""
    B, T = 4, 60
    cond, gt = mel_inputs(B, T, 71)
    with training():
        diff = package_diffusion("w64")
        opt = torch.optim.AdamW(diff.parameters(), lr=1e-3)
        losses, keys = [], []
        for _ in range(4):
            opt.zero_grad()
            torch.manual_seed(72)                                   # the same draws every step
            loss = diff(cond, gt_spec=gt, infer=False, k_step=100)
            loss.backward()
            keys.append(diff.denoise_fn.__dict__["_packed"][0])
            opt.step()
            losses.append(loss.item())
    assert len(set(keys)) == len(keys)
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


# ---- end to end: a diffusion-new.yaml step from package parts ------------------------------------------------------------
def test_diffusion_new_yaml_step_from_package_parts():
    """Unit2Wav's training step (diffusion/vocoder.py): CombSubFast(infer=False) with its own PCmer Unit2Control ->
    get_mel -> F.mse_loss(ddsp_mel, gt) plus GaussianDiffusion(hidden, gt, k_step=100, infer=False) around
    WaveNet(128, 20, 512, 256), backward.  At the first step: the diffusion loss, the WaveNet's gradients and the hidden
    output's cotangent against float64 autograd of the oracle fed the step's own hidden output and draws; the control
    network's gradients against the float64 oracle network fed the step's inputs and output cotangents (the synthesizer's
    and get_mel's backwards have their own tests against the oracle port).  Then AdamW steps lower the loss and repack
    both networks' weights."""
    from tests.test_gpu_u2c_pcmer_backward import _capture, _check_against_oracle, _oracle_grads
    from ddsp_svc_b200 import synthetic as syn
    SR, P, B, nF = 44100, 512, 2, 40
    torch.manual_seed(81)
    model = pkg.CombSubFast(SR, P, n_unit=768, n_spk=2, use_pitch_aug=True)
    model.unit2ctrl.pcmer_backward = True
    model = model.to(DEV).train()
    diff = package_diffusion("w512").train()
    diff.denoise_fn.diffusion_backward = True
    g = torch.Generator().manual_seed(82)
    dev = lambda x: x.to(DEV)
    f0 = dev(syn.make_f0(B, nF, SR, P, seed=83))
    units, volume = dev(torch.randn(B, nF, 768, generator=g)), dev(0.2 * torch.rand(B, nF, 1, generator=g))
    spk, aug = dev(torch.LongTensor([[2], [1]])), dev(torch.tensor([[[1.5]], [[-2.0]]]))
    noise = dev(syn.uniform_noise(B, nF * P, 84))
    stft = pkg.mel.STFT(SR, 128, 2048, 2048, P, 40, 16000)
    with torch.no_grad():
        sig0, _, _ = model(units, f0, volume, spk_id=spk, aug_shift=aug, noise=noise)
        mel0 = stft.get_mel(sig0).transpose(1, 2)
    gt = (mel0 + 0.5 * torch.randn(mel0.shape, generator=g).to(DEV)).contiguous()
    assert gt.shape == (B, nF, 128)
    seen = _capture(model.unit2ctrl)
    opt = torch.optim.AdamW(list(model.parameters()) + list(diff.parameters()), lr=2e-4)
    losses, packs = [], []
    for step in range(4):
        opt.zero_grad()
        signal, hidden, _ = model(units, f0, volume, spk_id=spk, aug_shift=aug, infer=False, noise=noise)
        ddsp_mel = stft.get_mel(signal).transpose(1, 2)
        torch.manual_seed(85)                                       # the same draws every step
        diff_loss = diff(hidden, gt_spec=gt, k_step=100, infer=False)
        loss = torch.nn.functional.mse_loss(ddsp_mel, gt) + diff_loss
        loss.backward()
        packs.append((model.unit2ctrl.__dict__["_packed"][0], diff.denoise_fn.__dict__["_packed"][0]))
        if step == 0:
            for n, p in diff.denoise_fn.named_parameters():
                assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().max() > 0, n
            torch.manual_seed(85)
            t, nz = DG.draws(B, nF, 100, device=DEV)
            loss64, want = oracle_gradients("w512", seen["h"].detach(), gt, t, nz)
            got = {n: p.grad for n, p in diff.denoise_fn.named_parameters()}
            got["condition"] = seen["h"].grad
            errs = {n: rel(got[n], w) for n, w in want.items()}
            errs["loss"] = rel(diff_loss, loss64)
            report.record("diffusion_backward/e2e_first_step/wavenet", **errs)
            params = {n: e for n, e in errs.items() if n != "condition"}
            assert max(params.values()) <= NETWORK_BOUND["3xtf32"], params
            assert errs["condition"] <= CONDITION_BOUND["3xtf32"], errs["condition"]
            kw = dict(use_pitch_aug=True)
            want_u = _oracle_grads(model.unit2ctrl, seen, **kw)
            want32_u = _oracle_grads(model.unit2ctrl, seen, torch.float32, **kw)
            got_u = {n: p.grad for n, p in model.unit2ctrl.named_parameters()}
            assert all((got_u[n] is None) == (w is None) for n, w in want_u.items())
            _check_against_oracle(got_u, want_u, want32_u, "diffusion_backward/e2e_first_step/unit2control")
        opt.step()
        losses.append(loss.item())
    report.record("diffusion_backward/e2e_adamw", first=losses[0], last=losses[-1])
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    assert len(set(p[0] for p in packs)) == len(packs) and len(set(p[1] for p in packs)) == len(packs)
