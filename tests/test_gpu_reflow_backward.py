"""The reflow loss and the velocity network's CUDA backward (csrc/reflow_bwd.cu + library GEMMs, ddsp_svc_b200/reflow.py
and denoiser.py: _LossFunction, _NetworkFunction) on the GPU:

* the reference's own loss and float64 gradients replayed (tests/golden/reflow_grad_*.npz) in the three GEMM modes;
* the 512-wide, 6-layer network of configs/reflow.yaml at its training batch (48 x 172) and at 1 x 861, against float64
  autograd of the oracle (tests/reflow_oracle.py) on the same GPU;
* each new kernel alone through the C ABI against float64, run twice (bit-identical);
* the training forward is the no_grad forward, determinism, the reference's draws, refusals;
* end to end: a configs/reflow.yaml step from package parts (CombSubSuperFast with its own Unit2Control -> get_mel ->
  mse + reflow loss -> backward) against the oracle chain, then AdamW steps.

Errors are relative RMS against float64 per tensor, recorded through tests/report.py (B2D_PARITY_REPORT)."""
import contextlib
import json

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import _lib, ops, synthetic as syn
from ddsp_svc_b200 import mel as pm
from ddsp_svc_b200.unit2control import Unit2Control
from tests import report, util
from tests.golden import make_golden_reflow as mk
from tests.golden import make_golden_reflow_grad as GR

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MODES = ("3xtf32", "fp32", "tf32")
# Bounds are about 3 times the largest error measured on an H100 80GB HBM3 at 700 W (DESIGN.md section 4.14b).
# Fixtures (w128, the stored entries): each tensor within max(3 err32, floor), err32 the reference's own fp32 error.
# Measured worst tensors: fp32 9.1e-6 and 3xtf32 9.6e-6 (diffusion_embedding.3.weight: the step MLP's B-row products,
# which the reference's own fp32 run misses by 6e-6 to 1.2e-5), tf32 1.3e-3 (condition: one TF32 pass rounds every operand to 11 bits, 4.9e-4 relative, and the
# condition's cotangent goes through every layer's forward and backward products).  Loss: 1.9e-6 / 1.5e-7 / 9.2e-5.
FIXTURE_FLOOR = {"fp32": 3e-5, "3xtf32": 3e-5, "tf32": 4e-3}
# the w512 network against float64, worst tensor and the loss: fp32 3.6e-6, 3xtf32 3.2e-5 (48 x 172; 2.7e-5 at
# 1 x 861), tf32 2.5e-3
NETWORK_BOUND = {"fp32": 1e-5, "3xtf32": 1e-4, "tf32": 8e-3}


def rel(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return util.rms(got - want) / max(util.rms(want), 1e-300)


@contextlib.contextmanager
def training(mode="3xtf32"):
    prev = pkg.NaiveV2Diff.gemm_precision, pkg.NaiveV2Diff.reflow_backward
    pkg.NaiveV2Diff.gemm_precision, pkg.NaiveV2Diff.reflow_backward = mode, True
    try:
        yield
    finally:
        pkg.NaiveV2Diff.gemm_precision, pkg.NaiveV2Diff.reflow_backward = prev


def package_flow(model):
    net = pkg.NaiveV2Diff(use_mlp=False, **mk.model_kwargs(model))
    net.load_state_dict(mk.build_oracle(model).state_dict(), strict=True)
    return pkg.RectifiedFlow(net.to(DEV))


def draws(B, T, seed, t_start=0.0, M=128):
    """the reference's draws on the device under torch.manual_seed(seed)"""
    torch.manual_seed(seed)
    t = torch.clip(t_start + (1.0 - t_start) * torch.rand(B, device=DEV), 1e-7, 1 - 1e-7)
    x0 = torch.empty_strided((B, 1, M, T), (T * M, T * M, 1, M), device=DEV).normal_()
    return t, x0[:, 0].transpose(1, 2)


def mel_inputs(B, T, seed, M=128):
    g = torch.Generator().manual_seed(seed)
    ramp = torch.linspace(-8.0, 0.5, M)[None, None, :]
    return ((ramp + 1.5 * torch.randn(B, T, M, generator=g)).to(DEV),
            (ramp + 1.5 * torch.randn(B, T, M, generator=g)).to(DEV))


def package_gradients(flow, cond, gt, t, x0):
    flow.zero_grad(set_to_none=True)
    c = cond.clone().requires_grad_(True)
    loss = flow._loss(c, gt, t, x0)
    loss.backward()
    grads = {n: p.grad for n, p in flow.velocity_fn.named_parameters()}
    grads["condition"] = c.grad
    return loss.detach(), grads


def oracle_gradients(model, cond, gt, t, x0, dtype=torch.float64):
    net = mk.build_oracle(model).to(DEV, dtype)
    c = cond.to(dtype).clone().requires_grad_(True)
    loss = GR.oracle_loss(net, c, gt, t, x0)
    loss.backward()
    grads = {n: p.grad for n, p in net.named_parameters()}
    grads["condition"] = c.grad
    return loss.detach(), grads


# ---- the reference's gradients replayed ----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(GR.CASES))
def test_fixture_loss_and_gradients(name, mode):
    d = np.load(GR.path(name))
    dev = lambda k: torch.from_numpy(d[k]).to(DEV)
    with training(mode):
        flow = package_flow(GR.MODEL)
        loss, grads = package_gradients(flow, dev("condition"), dev("gt_spec"), dev("t"), dev("x0"))
    loss64, loss32 = float(d["loss64"]), float(d["loss32"])
    loss_err, ref_loss_err = abs(loss.item() - loss64) / loss64, abs(loss32 - loss64) / loss64
    errs, over = {}, {}
    assert {n for n, g in grads.items() if g is None} == set(json.loads(str(d["none"])))    # the unused LayerNorms
    for n, g in GR.stored(name, grads).items():                    # the entries the fixture keeps
        errs[n] = rel(g, torch.from_numpy(d["f64/" + n]))
        bound = max(3 * float(d["err32/" + n]), FIXTURE_FLOOR[mode])
        if not errs[n] <= bound:
            over[n] = (errs[n], bound)
    report.record("reflow_backward/fixture/%s/%s" % (name, mode), loss=loss_err, ref32_loss=ref_loss_err,
                  max_grad=max(errs.values()), **errs)
    assert loss_err <= max(3 * ref_loss_err, FIXTURE_FLOOR[mode]), (loss_err, ref_loss_err)
    assert not over, over


# ---- the reflow.yaml network against float64 -----------------------------------------------------------------------------
@pytest.mark.parametrize("mode,B,T", [("3xtf32", 48, 172), ("fp32", 48, 172), ("tf32", 48, 172), ("3xtf32", 1, 861)])
def test_reflow_network_gradients_against_float64(mode, B, T):
    cond, gt = mel_inputs(B, T, B + T)
    t, x0 = draws(B, T, 7 + B, t_start=0.0)
    with training(mode):
        flow = package_flow("w512")
        loss, grads = package_gradients(flow, cond, gt, t, x0)
    loss64, want = oracle_gradients("w512", cond, gt, t, x0)
    errs = {n: rel(g, want[n]) for n, g in grads.items() if want[n] is not None}
    assert all(grads[n] is None for n, w in want.items() if w is None)
    report.record("reflow_backward/w512/%s/%dx%d" % (mode, B, T), loss=rel(loss, loss64), max_grad=max(errs.values()),
                  **errs)
    bound = NETWORK_BOUND[mode]
    assert rel(loss, loss64) <= bound
    assert max(errs.values()) <= bound, {n: e for n, e in errs.items() if e > bound}


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


@pytest.mark.parametrize("B,T", [(48, 172), (32, 861)])
def test_loss_kernels(B, T):
    L, M, st = _lib.lib(), 128, ops._stream()
    gt, x0, g, bias = _rand(B, T, M, seed=1, scale=3), _rand(B, T, M, seed=2), _rand(B, T, M, seed=3), _rand(M, seed=4)
    t = torch.clip(torch.rand(B, generator=torch.Generator().manual_seed(5)), 1e-7, 1 - 1e-7).to(DEV)
    w = 0.398942 / t / (1 - t) * torch.exp(-0.5 * torch.log(t / (1 - t)) ** 2)
    gl = torch.tensor([0.6], device=DEV)
    n = L.b2d_rf_backward_workspace_bytes(B, T, M)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)

    def run():
        target, hi, lo, loss = _nan(B, T, M), _nan(B, T, M), _nan(B, T, M), _nan(1)
        gv, ghi, glo = _nan(B, T, M), _nan(B, T, M), _nan(B, T, M)
        _lib.check(L.b2d_rf_loss_input(gt.data_ptr(), x0.data_ptr(), t.data_ptr(), -12.0, 14.0, B, T, M, target.data_ptr(),
                                       hi.data_ptr(), lo.data_ptr(), st), "rf_loss_input")
        _lib.check(L.b2d_rf_loss(g.data_ptr(), bias.data_ptr(), target.data_ptr(), w.data_ptr(), B, T, M, ws.data_ptr(), n,
                                 loss.data_ptr(), st), "rf_loss")
        _lib.check(L.b2d_rf_loss_backward(g.data_ptr(), bias.data_ptr(), target.data_ptr(), w.data_ptr(), gl.data_ptr(), B, T,
                                          M, gv.data_ptr(), ghi.data_ptr(), glo.data_ptr(), st), "rf_loss_backward")
        return target, hi, lo, loss, gv, ghi, glo

    target, hi, lo, loss, gv, ghi, glo = _twice(run)
    d = lambda x: x.double()
    x1 = (d(gt) + 12) / 14 * 2 - 1
    e = {"target": rel(target, x1 - d(x0)), "x_t": rel(d(hi) + d(lo), d(x0) + d(t)[:, None, None] * (x1 - d(x0)))}
    r = d(target) - (d(g) + d(bias))
    want_loss = (d(w)[:, None, None] * r * r).mean()
    e["loss"] = abs(loss.double().item() - want_loss.item()) / want_loss.item()
    want_gv = -0.6 * 2 * d(w)[:, None, None] * r / r.numel()
    e["gv"], e["gv_halves"] = rel(gv, want_gv), rel(d(ghi) + d(glo), want_gv)
    report.record("reflow_backward/kernels/loss/%dx%d" % (B, T), **e)
    assert max(e.values()) <= 1e-6, e


@pytest.mark.parametrize("B,T", [(48, 172), (32, 861)])
def test_gelu_and_layer_backward_kernels(B, T):
    L, D, nL, st = _lib.lib(), 512, 6, ops._stream()
    N, LD = B * T, 512 * 6
    gy, pre, bias = _rand(N, D, seed=11), _rand(N, D, seed=12, scale=2), _rand(D, seed=13)
    gz = [_rand(N, D, seed=20 + i) for i in range(nL)]
    gh0 = _rand(N, D, seed=14)
    n = L.b2d_rf_backward_workspace_bytes(B, T, LD)
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)

    def run():
        gx, hi, lo = _nan(N, D), _nan(N, D), _nan(N, D)
        _lib.check(L.b2d_rf_gelu_backward(gy.data_ptr(), pre.data_ptr(), bias.data_ptr(), N, D, gx.data_ptr(), hi.data_ptr(),
                                          lo.data_ptr(), st), "rf_gelu_backward")
        gh, hh, hl, z, zh, zl, gS = gh0.clone(), _nan(N, D), _nan(N, D), _nan(N, LD), _nan(N, LD), _nan(N, LD), _nan(B, LD)
        for i in reversed(range(nL)):
            _lib.check(L.b2d_rf_layer_backward(gz[i].data_ptr(), gh.data_ptr(), B, T, D, i, nL, hh.data_ptr(), hl.data_ptr(),
                                               z.data_ptr(), zh.data_ptr(), zl.data_ptr(), ws.data_ptr(), n, st),
                       "rf_layer_backward")
        _lib.check(L.b2d_rf_step_sums(ws.data_ptr(), n, B, T, LD, gS.data_ptr(), st), "rf_step_sums")
        return gx, hi, lo, gh, hh, hl, z, zh, zl, gS

    gx, hi, lo, gh, hh, hl, z, zh, zl, gS = _twice(run)
    x = (pre.double() + bias.double()).requires_grad_(True)
    torch.nn.functional.gelu(x).backward(gy.double())
    d = lambda v: v.double()
    want_h = d(gh0) + sum(d(v) for v in gz)
    want_z = torch.cat([d(v) for v in gz], dim=1)
    e = {"gelu": rel(gx, x.grad), "gelu_halves": rel(d(hi) + d(lo), x.grad), "gh": rel(gh, want_h),
         "gh_halves": rel(d(hh) + d(hl), want_h), "z_halves": rel(d(zh) + d(zl), want_z),
         "step_sums": rel(gS, want_z.reshape(B, T, LD).sum(1))}
    assert torch.equal(z, want_z.float())
    report.record("reflow_backward/kernels/layer/%dx%d" % (B, T), **e)
    assert max(e.values()) <= 1e-6, e


# ---- the training forward, determinism, draws, refusals ------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_training_forward_is_the_no_grad_forward(mode):
    B, T = 3, 70
    cond, gt = mel_inputs(B, T, 31)
    spec = torch.randn(B, 128, T, generator=torch.Generator().manual_seed(32)).to(DEV)
    steps = torch.tensor([10.0, 500.0, 990.0], device=DEV)
    t, x0 = draws(B, T, 33)
    with training(mode):
        flow = package_flow("w512")
        net = flow.velocity_fn
        with torch.no_grad():
            v0 = net(spec[:, None], steps, cond.transpose(1, 2))
            l0 = flow._loss(cond, gt, t, x0)
        v1 = net(spec[:, None], steps, cond.transpose(1, 2))
        l1 = flow._loss(cond, gt, t, x0)
        c = cond.clone().requires_grad_(True)
        net.requires_grad_(False)
        v2 = net(spec, steps, c.transpose(1, 2))                  # only cond requires grad
        l2 = flow._loss(c, gt, t, x0)
    assert v1.requires_grad and l1.requires_grad and v2.requires_grad and l2.requires_grad and not v0.requires_grad
    assert torch.equal(v0, v1) and torch.equal(v0[:, 0], v2) and torch.equal(l0, l1) and torch.equal(l0, l2)


def test_two_backwards_and_two_runs_are_bit_identical():
    B, T = 4, 150
    cond, gt = mel_inputs(B, T, 41)
    t, x0 = draws(B, T, 42)
    with training():
        flow = package_flow("w512")
        params = [p for n, p in flow.velocity_fn.named_parameters() if ".norm." not in n]
        c = cond.clone().requires_grad_(True)
        loss = flow._loss(c, gt, t, x0)
        a = torch.autograd.grad(loss, params + [c], retain_graph=True)
        b = torch.autograd.grad(loss, params + [c])
        c2 = cond.clone().requires_grad_(True)
        d = torch.autograd.grad(flow._loss(c2, gt, t, x0), params + [c2])
        spec, steps = x0.transpose(1, 2).contiguous(), 1000 * t
        cot = torch.randn(B, 128, T, generator=torch.Generator().manual_seed(43)).to(DEV)
        e = torch.autograd.grad((flow.velocity_fn(spec, steps, c.transpose(1, 2)) * cot).sum(), params + [c])
        f = torch.autograd.grad((flow.velocity_fn(spec, steps, c.transpose(1, 2)) * cot).sum(), params + [c])
    assert all(torch.equal(x, y) and torch.equal(x, z) for x, y, z in zip(a, b, d))
    assert all(torch.equal(x, y) for x, y in zip(e, f))


def test_seeded_draws_are_the_references_expressions():
    """forward(infer=False) under a seed equals _loss fed the reference's own expressions: t from torch.rand, then x_0 =
    torch.randn_like of the transposed [B, 1, M, T] view of norm(gt_spec) (reflow/reflow.py:64-67, :21)"""
    B, T = 3, 50
    cond, gt = mel_inputs(B, T, 51)
    with training():
        flow = package_flow("w128")
        with torch.no_grad():
            torch.manual_seed(52)
            a = flow(cond, gt_spec=gt, infer=False, t_start=0.7)
            torch.manual_seed(52)
            t = torch.clip(0.7 + (1.0 - 0.7) * torch.rand(B, device=DEV), 1e-7, 1 - 1e-7)
            x1 = ((gt - (-12)) / (2 - (-12)) * 2 - 1).transpose(1, 2)[:, None, :, :]
            x0 = torch.randn_like(x1)
            b = flow._loss(cond, gt, t, x0[:, 0].transpose(1, 2))
            torch.manual_seed(52)
            c = flow(cond, gt_spec=gt, infer=False, t_start=0.7)
            torch.manual_seed(53)
            e = flow(cond, gt_spec=gt, infer=False, t_start=0.7)
        torch.manual_seed(52)
        f = flow(cond, gt_spec=gt, infer=False, t_start=0.7)        # under grad: the same value
    assert torch.equal(a, b) and torch.equal(a, c) and not torch.equal(a, e) and torch.equal(a, f.detach())
    assert x0.stride(0) == T * 128 and x0.stride()[2:] == (1, 128)           # token-major (dim 1 has size 1)


def test_switch_and_refusals():
    assert pkg.NaiveV2Diff.reflow_backward is False
    flow = package_flow("w128")
    cond, gt = mel_inputs(2, 20, 61)
    t, x0 = draws(2, 20, 62)
    with pytest.raises(NotImplementedError, match="training"):
        flow(cond, gt_spec=gt, infer=False)
    with pytest.raises(NotImplementedError, match="training"):
        flow.velocity_fn(x0.transpose(1, 2), 1000 * t, cond.transpose(1, 2))
    flow.velocity_fn.reflow_backward = True                         # per instance
    loss = flow(cond, gt_spec=gt, infer=False)
    assert loss.requires_grad and loss.dim() == 0
    with pytest.raises(NotImplementedError, match="not differentiable"):
        flow(cond, gt_spec=gt, infer=True)
    with pytest.raises(NotImplementedError, match="spec"):
        flow.velocity_fn(x0.transpose(1, 2).clone().requires_grad_(True), 1000 * t, cond.transpose(1, 2))
    with pytest.raises(NotImplementedError, match="l1"):
        flow._loss(cond, gt, t, x0, loss_type="l1")
    with pytest.raises(NotImplementedError, match="data"):
        flow._loss(cond, gt.clone().requires_grad_(True), t, x0)
    with pytest.raises(ValueError, match="gt_spec"):
        flow(cond, gt_spec=None, infer=False)
    assert pkg.NaiveV2Diff.reflow_backward is False
    with torch.no_grad():
        flow(cond, gt_spec=gt, infer_step=1)                        # the sampler still runs without grad


# ---- end to end: a reflow.yaml step from package parts --------------------------------------------------------------------
def test_reflow_yaml_step_from_package_parts():
    """CombSubSuperFast (its own Unit2Control) -> get_mel -> F.mse_loss(ddsp_mel, gt) + RectifiedFlow(infer=False)
    (reflow/vocoder.py:177-186), backward: every parameter of both networks gets a gradient.  At the first step the
    gradients are compared with the oracle chain (oracle control network + oracle.torch_port + oracle.mel in fp32 on the
    CPU, the reflow oracle in float64) fed the same draws; then AdamW steps lower the loss and repack the weights."""
    from oracle import mel as om
    from oracle import torch_port as tp
    from oracle.unit2control import NaiveUnit2Control
    SR, P, WIN, B, nF = 44100, 512, 2048, 2, 40
    torch.manual_seed(71)
    model = pkg.CombSubSuperFast(SR, P, WIN, n_unit=768, n_spk=2, use_pitch_aug=True)
    assert isinstance(model.unit2ctrl, Unit2Control) and model.unit2ctrl.use_naive_v2
    u2c_oracle = NaiveUnit2Control(768, 2, model.unit2ctrl.output_splits, use_pitch_aug=True).train()
    u2c_oracle.load_state_dict(model.unit2ctrl.state_dict())
    model = model.to(DEV).train()
    flow = package_flow("w512").train()
    flow.velocity_fn.reflow_backward = True
    g = torch.Generator().manual_seed(72)
    f0 = syn.make_f0(B, nF, SR, P, seed=73)
    units, volume = torch.randn(B, nF, 768, generator=g), 0.2 * torch.rand(B, nF, 1, generator=g)
    spk, aug = torch.LongTensor([[2], [1]]), torch.tensor([[[1.5]], [[-2.0]]])
    noise = syn.normal_noise((B, nF * P), 74)
    stft = pm.STFT(SR, 128, 2048, 2048, P, 40, 16000)
    dev = lambda x: x.to(DEV)
    with torch.no_grad():
        sig0, _, _ = model(dev(units), dev(f0), dev(volume), spk_id=dev(spk), aug_shift=dev(aug), noise=dev(noise))
        mel0 = stft.get_mel(sig0).transpose(1, 2)
    gt = (mel0 + 0.5 * torch.randn(mel0.shape, generator=g).to(DEV)).contiguous()
    Tm = gt.shape[1]
    params = list(model.parameters()) + list(flow.parameters())
    opt = torch.optim.AdamW(params, lr=2e-4)
    losses, packs = [], []
    for step in range(4):
        opt.zero_grad()
        signal, _, _ = model(dev(units), dev(f0), dev(volume), spk_id=dev(spk), aug_shift=dev(aug), infer=False,
                             noise=dev(noise))
        ddsp_mel = stft.get_mel(signal).transpose(1, 2)             # reflow/vocoder.py extract(): [B, F, n_mels]
        torch.manual_seed(75)                                       # the same draws every step
        loss = torch.nn.functional.mse_loss(ddsp_mel, gt) + flow(ddsp_mel, gt_spec=gt, infer=False, t_start=0.0)
        loss.backward()
        packs.append((model.unit2ctrl.__dict__["_packed"][0], flow.velocity_fn.__dict__["_packed"][0]))
        if step == 0:
            named = [("u2c." + n, p) for n, p in model.unit2ctrl.named_parameters()] + \
                    [("vel." + n, p) for n, p in flow.velocity_fn.named_parameters()]
            for n, p in named:
                if ".norm." in n and (n.startswith("vel.residual_layers") or n.startswith("u2c.decoder")):
                    assert p.grad is None, n
                else:
                    assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().max() > 0, n
            t, x0 = draws(B, Tm, 75)
            with torch.no_grad():
                _, phase = ops.superfast_scan(dev(f0), P, SR)
            ctrls, _ = u2c_oracle(units, f0, phase.cpu().reshape(B, nF, 1), volume, spk_id=spk, aug_shift=aug)
            sig = tp.superfast_forward(f0, ctrls, SR, P, WIN, noise=noise)["signal"]
            m = om.get_mel(sig).transpose(1, 2)
            vel = mk.build_oracle("w512").double()
            ref_loss = torch.nn.functional.mse_loss(m, gt.cpu()) + GR.oracle_loss(vel, m.double(), gt.cpu(), t.cpu(), x0.cpu())
            ref_loss.backward()
            errs = {"loss": rel(loss, ref_loss)}
            oracle_params = dict([("u2c." + n, q) for n, q in u2c_oracle.named_parameters()] +
                                 [("vel." + n, q) for n, q in vel.named_parameters()])
            for n, p in named:
                if oracle_params[n].grad is not None:
                    errs[n] = rel(p.grad, oracle_params[n].grad)
            report.record("reflow_backward/e2e_first_step", **errs)
            # measured 2.9e-5 at worst (u2c.phase_embed.weight; the velocity network's tensors up to 7.0e-6)
            assert max(errs.values()) <= 1e-4, {n: e for n, e in errs.items() if e > 1e-4}
        opt.step()
        losses.append(loss.item())
    report.record("reflow_backward/e2e_adamw", first=losses[0], last=losses[-1])
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    assert len(set(p[0] for p in packs)) == len(packs) and len(set(p[1] for p in packs)) == len(packs)
