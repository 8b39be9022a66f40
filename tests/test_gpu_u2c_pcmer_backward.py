"""The CUDA backward of Unit2Control with the PCmer decoder (``Unit2Control.pcmer_backward``: csrc/pcmer_bwd.cu +
csrc/unit2control_bwd.cu + library GEMMs, ddsp_svc_b200/unit2control.py: _Unit2ControlFunction) on the GPU:

* each new kernel alone through the C ABI against a float64 torch expression at the rows of 24 x 172 and 32 x 861, run
  twice into NaN-filled outputs (finite, bit-identical);
* every parameter gradient of the whole module against the reference's own float64 gradients
  (tests/golden/u2c_pcmer_grad_*.npz) in the three GEMM modes and both fused_attention settings, and against the float64
  oracle (tests/u2c_pcmer_oracle.py: PCmerUnit2Control) at the training batch;
* determinism, per-utterance sums, forward identity with the no_grad call, launch counts, frozen parameters, refusals;
* end to end: the sins.yaml step (Sins with its own Unit2Control + RSSLoss, then AdamW), CombSubFast with pcmer_norm
  through the mel loss of DiffusionNew, and one CombSub (old) step."""
import json

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import _lib, ops, synthetic as syn
from ddsp_svc_b200.unit2control import Unit2Control
from tests import report, util
from tests.golden import make_golden_u2c_pcmer_grad as GP
from tests.test_emu_u2c_pcmer_backward import (features, features_backward_reference, qkv_gather_reference,
                                               readout_backward_reference)
from tests.u2c_pcmer_oracle import PCmerUnit2Control

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(24, 172), (32, 861)]
H, J = 8, 266


def _rel(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return util.rms(got - want) / max(util.rms(want), 1e-300)


def _rand(*shape, seed, scale=1.0):
    return (scale * torch.randn(*shape, generator=torch.Generator().manual_seed(seed))).to(DEV)


def _twice(fn):
    """run a kernel call twice into fresh NaN-filled outputs: the results must be finite and bit-identical"""
    a, b = fn(), fn()
    for x, y in zip(a, b):
        assert torch.isfinite(x).all() and torch.equal(x, y)
    return a


# ---- the kernels alone ----
@pytest.mark.parametrize("B,T", SHAPES)
def test_readout_backward_kernel(B, T):
    g_out, out = _rand(B, T, H, 64, seed=1), _rand(B, T, H, 64, seed=2)
    d_inv = 0.1 + _rand(B, H, T, seed=3).abs()

    def run():
        gn = torch.full((B, H, T, 65), np.nan, device=DEV)
        _lib.check(_lib.lib().b2d_u2c_attn_readout_backward(g_out.data_ptr(), out.data_ptr(), d_inv.data_ptr(), B, H, T, 64,
                                                            gn.data_ptr(), 0), "readout backward")
        return (gn,)

    e = _rel(_twice(run)[0], readout_backward_reference(g_out, out, d_inv))
    report.record("u2c_pcmer_backward/readout/%dx%d" % (B, T), err=e)
    assert e <= 2e-6


@pytest.mark.parametrize("is_query", [1, 0])
@pytest.mark.parametrize("B,T", SHAPES)
def test_feature_backward_kernel(B, T, is_query):
    R = B * H * T
    dd, x = _rand(R, J, seed=4, scale=2.0), _rand(R, 64, seed=5, scale=0.5)
    phi = features(dd, x, is_query)
    gphi, vec, scal = _rand(R, J, seed=6), _rand(B * H, J, seed=7).abs(), _rand(R, seed=8)

    def run():
        g, gx = gphi.clone(), torch.full((R, 64), np.nan, device=DEV)
        _lib.check(_lib.lib().b2d_u2c_softmax_features_backward(g.data_ptr(), phi.data_ptr(), x.data_ptr(), vec.data_ptr(),
                                                                scal.data_ptr(), R, T, J, 64, is_query, 1e-4, gx.data_ptr(), 0),
                   "feature backward")
        return g, gx

    g, gx = _twice(run)
    want_dd, want_x = features_backward_reference(gphi, dd, x, vec, scal, T, is_query)
    e = dict(g_dd=_rel(g, want_dd), g_x=_rel(gx, want_x))
    report.record("u2c_pcmer_backward/features/%dx%d_q%d" % (B, T, is_query), **e)
    assert max(e.values()) <= 2e-6, e


@pytest.mark.parametrize("normalized", [0, 1])
@pytest.mark.parametrize("B,T", SHAPES)
def test_qkv_gather_backward_kernel(B, T, normalized):
    gq, gk, gv = _rand(B, H, T, 64, seed=9), _rand(B, H, T, 64, seed=10), _rand(B, H, T, 64, seed=11)
    qkv = _rand(B, T, 3, H, 64, seed=12, scale=3.0)

    def run():
        out = torch.full((B, T, 3, H, 64), np.nan, device=DEV)
        _lib.check(_lib.lib().b2d_u2c_qkv_gather_backward(gq.data_ptr(), gk.data_ptr(), gv.data_ptr(), qkv.data_ptr(), B, H, T, 64,
                                                          normalized, out.data_ptr(), 0), "qkv gather backward")
        return (out,)

    e = _rel(_twice(run)[0], qkv_gather_reference(gq, gk, gv, qkv, normalized))
    report.record("u2c_pcmer_backward/qkv_gather/%dx%d_n%d" % (B, T, normalized), err=e)
    assert e <= 2e-6


# ---- the whole module ----
# 3xtf32: 2e-5 as for the convolution-only decoder, or 3x the reference's own fp32 error where that is larger.  The query
# side's cotangent (g_num ctx^T + g_D ksum, then the feature map's row sums) cancels, so fp32 rounding is amplified there:
# the reference's own fp32 gradients of to_q measure 1.0e-5 to 4.1e-5 against float64 on the goldens without pcmer_norm
# and 1.9e-4 with it, and the kernels at 3xtf32 measured 2.4e-5 on to_q of layer 0 at 768 units (H100 SXM, 700 W).
BOUND = {"3xtf32": 2e-5, "tf32": 5e-3}
# Single-pass TF32 only, measured on an H100 SXM at 700 W: the tensors behind the convolution stack's LeakyReLU measure 8e-3
# to 2.2e-2 (a flipped LeakyReLU element, as for the convolution-only decoder: tests/test_gpu_unit2control_backward.py);
# the query / key projections 1.4e-3 to 1.3e-2 (the per-head products run in TF32 in this mode, as in the forward, and
# the cancellation above amplifies their rounding as it amplifies fp32's); every other tensor stays under 5e-3.
QK = (".attn.to_q.", ".attn.to_k.")


def _tf32_bound(n):
    return 5e-2 if n.startswith("stack.") else 3e-2 if any(q in n for q in QK) else BOUND["tf32"]


def _model(name, mode="3xtf32", fused=False):
    m = GP.build_model(name).to(DEV).train()
    m.gemm_precision, m.fused_attention, m.pcmer_backward = mode, fused, True
    return m


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("mode", ["fp32", "3xtf32", "tf32"])
@pytest.mark.parametrize("name", list(GP.CASES))
def test_parameter_gradients_match_the_reference(name, mode, fused):
    """each tensor within 3x the fp32 reference's own error against float64, with a floor of 1e-6 (fp32 GEMMs), 2e-5
    (3xtf32) or 5e-3 (tf32; _tf32_bound).  Relative RMS over the entries the golden stores."""
    gold = np.load(GP.path(name))
    grads = GP.gradients(_model(name, mode, fused), GP.build_inputs(name), torch.float32)
    assert {n for n, g in grads.items() if g is None} == set(json.loads(str(gold["none"])))
    errs, over = {}, {}
    for n, got in GP.stored(name, grads).items():
        want = gold["f64/" + n]
        errs[n] = util.rms(got.double().numpy() - want) / util.rms(want)
        floor = {"fp32": 1e-6, "3xtf32": BOUND["3xtf32"], "tf32": _tf32_bound(n)}[mode]
        bound = max(3 * float(gold["err32/" + n]), floor)
        if not errs[n] <= bound:
            over[n] = (errs[n], bound)
    report.record("u2c_pcmer_backward/module/%s/%s/fused%d" % (name, mode, fused), **errs)
    assert not over, over


@pytest.mark.parametrize("fused", [False, True])
def test_training_batch_gradients_match_the_float64_oracle(fused):
    """24 x 172 (the sins.yaml batch) at 768 units, default GEMM mode, every entry of every gradient"""
    name = "u2c_pcmer_grad_sins_spk3"
    B, T = 24, 172
    m = _model(name, fused=fused)
    g = torch.Generator().manual_seed(40)
    inp = dict(GP.build_inputs(name))
    inp.update(units=torch.randn(B, T, 768, generator=g), f0=220.0 * 2 ** (torch.rand(B, T, 1, generator=g) * 2 - 1),
               phase=torch.rand(B, T, 1, generator=g) * 6 - 3, volume=0.2 * torch.rand(B, T, 1, generator=g),
               spk_id=torch.randint(1, 4, (B, 1), generator=g), cot_dense=torch.randn(B, T, 640, generator=g),
               cot_hidden=torch.randn(B, T, 256, generator=g))
    inp["f0"][:, 30:40] = 0.0
    oracle = PCmerUnit2Control(**GP.model_kwargs(name)).train()
    oracle.load_state_dict(m.state_dict())
    want = GP.gradients(oracle.to(DEV).double(), inp, torch.float64)
    want32 = GP.gradients(oracle.float(), inp, torch.float32)
    got = GP.gradients(m, inp, torch.float32)
    assert all(got[n] is None for n, w in want.items() if w is None)
    _check_against_oracle(got, want, want32, "u2c_pcmer_backward/module/training_batch/fused%d" % fused)


def _check_against_oracle(got, want, want32, label):
    """each gradient within max(2e-5, 3x the fp32 oracle's own error) of the float64 oracle (see BOUND)"""
    errs, over = {}, {}
    for n, w in want.items():
        if w is not None:
            errs[n] = _rel(got[n], w)
            bound = max(BOUND["3xtf32"], 3 * _rel(want32[n], w))
            if not errs[n] <= bound:
                over[n] = (errs[n], bound)
    report.record(label, **errs)
    assert not over, over


def _small(stack=True, norm=False, **kw):
    torch.manual_seed(7)
    m = Unit2Control(64, 3, GP.SMALL, use_conv_stack=stack, use_pitch_aug=True, pcmer_norm=norm, **kw).to(DEV)
    m.pcmer_backward = True
    return m


def _call_inputs(B=3, T=100, seed=8):
    g = torch.Generator().manual_seed(seed)
    return dict(units=torch.randn(B, T, 64, generator=g).to(DEV), f0=(100 + 300 * torch.rand(B, T, 1, generator=g)).to(DEV),
                phase=torch.randn(B, T, 1, generator=g).to(DEV), volume=torch.rand(B, T, 1, generator=g).to(DEV),
                spk_id=torch.randint(1, 4, (B, 1), generator=g).to(DEV), aug_shift=torch.randn(B, 1, 1, generator=g).to(DEV))


@pytest.mark.parametrize("fused", [False, True])
def test_two_backwards_from_one_forward_are_bit_identical(fused):
    m, inp = _small(norm=True), _call_inputs()
    m.fused_attention = fused
    ctrls, hidden = m(**inp)
    dense = torch.cat(list(ctrls.values()), -1)
    params = [p for n, p in m.named_parameters()]
    cot = (torch.randn_like(dense), torch.randn_like(hidden))
    a = torch.autograd.grad((dense, hidden), params, cot, retain_graph=True)
    b = torch.autograd.grad((dense, hidden), params, cot)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_single_utterance_gradients_add_up_to_the_batch_gradient():
    m, inp = _small(), _call_inputs()
    m.gemm_precision = "fp32"
    B = inp["units"].shape[0]
    g = torch.Generator().manual_seed(9)
    cot = dict(cot_dense=torch.randn(B, 100, 40, generator=g), cot_hidden=torch.randn(B, 100, 256, generator=g))
    cpu = {k: v.cpu() for k, v in inp.items()}
    full = GP.gradients(m, dict(cpu, **cot), torch.float32)
    parts = [GP.gradients(m, {k: v[b:b + 1] for k, v in dict(cpu, **cot).items()}, torch.float32) for b in range(B)]
    errs = {n: _rel(sum(p[n].double() for p in parts), w) for n, w in full.items() if w is not None}
    report.record("u2c_pcmer_backward/utterance_sums", **errs)
    # 2e-6; the query / key projections 1e-4: fp32 GEMMs summing in another order, amplified by the query side's
    # cancellation (see BOUND)
    over = {n: e for n, e in errs.items() if e > (1e-4 if any(q in n for q in QK) else 2e-6)}
    assert not over, over


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("stack,launches", [(False, 5 + 3 * 4), (True, 6 + 3 * 4)])
def test_forward_under_grad_is_the_no_grad_forward(stack, launches, fused):
    """same kernels: bit-identical without the convolution stack; with it the GroupNorm statistics are accumulated with
    fp64 atomics, so two forwards may differ in the last bit.  fp32 GEMMs: embed + 3 x (GLU stage, 2 LayerNorms, 2 feature
    maps) + LayerNorm (+ GroupNorm), and the fused read-out kernel per layer when fused_attention is on"""
    m, inp = _small(stack), _call_inputs()
    m.gemm_precision, m.fused_attention = "fp32", fused
    launches += 3 * fused
    with torch.no_grad():
        m(**inp)                                                  # packs the weights
        n0 = ops.launches()
        c0, h0 = m(**inp)
        assert ops.launches() - n0 == launches
    n0 = ops.launches()
    c1, h1 = m(**inp)
    assert ops.launches() - n0 == launches and h1.requires_grad and all(v.requires_grad for v in c1.values())
    m.requires_grad_(False)
    n0 = ops.launches()
    c2, h2 = m(**inp)
    assert ops.launches() - n0 == launches
    assert not h2.requires_grad and not any(v.requires_grad for v in c2.values())
    for a, b in ((h0, h1), (h0, h2)) + tuple((c0[k], c1[k]) for k in c0):
        assert torch.equal(a, b) if not stack else _rel(a, b) <= 1e-6
    assert next(iter(c1.values())).stride(1) == m.n_out           # still views of one dense tensor


def test_inputs_are_data_and_the_switch_is_off_by_default():
    m, inp = _small(), _call_inputs()
    for k in ("units", "f0", "phase", "volume", "aug_shift"):
        with pytest.raises(NotImplementedError):
            m(**dict(inp, **{k: inp[k].clone().requires_grad_(True)}))
    with pytest.raises(NotImplementedError):
        m(**dict(inp, spk_mix_dict={1: 0.5, 2: 0.5}))
    with torch.no_grad():
        m(**dict(inp, spk_mix_dict={1: 0.5, 2: 0.5}))              # inference keeps it
    assert Unit2Control.pcmer_backward is False
    m.pcmer_backward = False
    c, h = m(**inp)
    assert not h.requires_grad and not any(v.requires_grad for v in c.values())


# ---- end to end ----
def _capture(u2c):
    """wrap u2c.forward so the step's control / hidden cotangents and the call's inputs can be read after backward"""
    seen, forward = {}, u2c.forward

    def f(*a, **k):
        c, h = forward(*a, **k)
        for v in list(c.values()) + [h]:
            v.retain_grad()
        seen.update(c=c, h=h, a=a, k=k)
        return c, h
    u2c.forward = f
    return seen


def _oracle_grads(u2c, seen, dtype=torch.float64, **kw):
    """oracle network on the CPU with the step's own inputs and output cotangents -> {name: gradient}"""
    oracle = PCmerUnit2Control(seen["a"][0].shape[-1], u2c.n_spk, u2c.output_splits, **kw).train()
    oracle.load_state_dict(u2c.state_dict())
    oracle = oracle.to(dtype)
    cpu = lambda t: None if t is None else (t.detach().cpu().to(dtype) if t.is_floating_point() else t.detach().cpu())
    units, f0, phase, volume = (cpu(t) for t in seen["a"][:4])
    ctrls, hid = oracle(units, f0, phase, volume, spk_id=cpu(seen["k"].get("spk_id")), aug_shift=cpu(seen["k"].get("aug_shift")))
    loss = sum((ctrls[k] * cpu(seen["c"][k].grad)).sum() for k in ctrls if seen["c"][k].grad is not None)
    if seen["h"].grad is not None:
        loss = loss + (hid * cpu(seen["h"].grad)).sum()
    loss.backward()
    return {n: p.grad for n, p in oracle.named_parameters()}


def test_sins_yaml_step_trains_its_own_pcmer_unit2control():
    """Sins(44100, 512, 128, 256, 256, n_unit=768, n_spk=2) -> RSSLoss(256, 2048, 4): the first step's network
    gradients against the float64 oracle network fed the step's own inputs and control cotangents (the synthesizer's and
    the loss's backwards have their own tests against the oracle port and oracle loss), then eight AdamW steps"""
    SR, P, B, nF = 44100, 512, 2, 40
    n_ffts = [700, 1500, 300, 1024]
    torch.manual_seed(31)
    model = pkg.Sins(SR, P, 128, 256, 256, n_unit=768, n_spk=2)
    assert isinstance(model.unit2ctrl, Unit2Control) and not model.unit2ctrl.use_naive_v2
    model.unit2ctrl.pcmer_backward = True
    model = model.to(DEV).train()
    seen = _capture(model.unit2ctrl)
    g = torch.Generator().manual_seed(32)
    f0 = syn.make_f0(B, nF, SR, P, seed=33)
    units, volume = torch.randn(B, nF, 768, generator=g), 0.2 * torch.rand(B, nF, 1, generator=g)
    spk = torch.LongTensor([[2], [1]])
    noise = syn.uniform_noise(B, nF * P, 34)
    target = syn.uniform_noise(B, nF * P, 35) * 0.05
    crit = pkg.RSSLoss(256, 2048, 4)
    opt = torch.optim.AdamW(model.parameters(), lr=2e-4)
    dev = lambda t: t.to(DEV)
    losses, packs = [], []
    for step in range(8):
        opt.zero_grad()
        signal, hidden, _ = model(dev(units), dev(f0), dev(volume), spk_id=dev(spk), infer=False, noise=dev(noise))
        loss = crit(signal, dev(target), n_ffts=n_ffts)
        loss.backward()
        packs.append(model.unit2ctrl.__dict__["_packed"][0])
        if step == 0:
            want, want32 = _oracle_grads(model.unit2ctrl, seen), _oracle_grads(model.unit2ctrl, seen, torch.float32)
            got = {n: p.grad for n, p in model.unit2ctrl.named_parameters()}
            assert all((got[n] is None) == (w is None) for n, w in want.items())
            _check_against_oracle(got, want, want32, "u2c_pcmer_backward/sins_step_first")
        opt.step()
        losses.append(loss.item())
    report.record("u2c_pcmer_backward/sins_step_adamw", first=losses[0], last=losses[-1])
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    assert len(set(packs)) == len(packs)                           # every step packed the weights the optimizer left


def test_combsubfast_pcmer_norm_trains_through_the_mel_loss():
    """the DDSP half of DiffusionNew (diffusion-new-fp16.yaml's pcmer_norm, pitch augmentation): CombSubFast ->
    STFT.get_mel -> MSE against a target mel; network gradients against the float64 oracle as above"""
    SR, P, B, nF = 44100, 512, 2, 32
    torch.manual_seed(41)
    model = pkg.CombSubFast(SR, P, n_unit=64, n_spk=2, use_pitch_aug=True, pcmer_norm=True)
    model.unit2ctrl.pcmer_backward = True
    model = model.to(DEV).train()
    seen = _capture(model.unit2ctrl)
    g = torch.Generator().manual_seed(42)
    f0 = syn.make_f0(B, nF, SR, P, seed=43)
    units, volume = torch.randn(B, nF, 64, generator=g), 0.2 * torch.rand(B, nF, 1, generator=g)
    stft = pkg.mel.STFT(SR, 128, 2048, 2048, 512, 40, 16000)
    target = torch.randn(B, 128, nF, generator=g).to(DEV) * 0.1 - 5
    dev = lambda t: t.to(DEV)
    signal, _, _ = model(dev(units), dev(f0), dev(volume), spk_id=dev(torch.LongTensor([[1], [2]])),
                         aug_shift=dev(torch.tensor([[[2.0]], [[-1.0]]])), infer=False, noise=dev(syn.uniform_noise(B, nF * P, 44)))
    mel = stft.get_mel(signal)
    loss = ((mel - target[..., :mel.shape[-1]]) ** 2).mean()
    loss.backward()
    kw = dict(use_pitch_aug=True, pcmer_norm=True)
    want, want32 = _oracle_grads(model.unit2ctrl, seen, **kw), _oracle_grads(model.unit2ctrl, seen, torch.float32, **kw)
    got = {n: p.grad for n, p in model.unit2ctrl.named_parameters()}
    assert all((got[n] is None) == (w is None) for n, w in want.items())
    _check_against_oracle(got, want, want32, "u2c_pcmer_backward/combsubfast_mel")


def test_combsub_old_step_reaches_every_unit2ctrl_parameter():
    SR, P, B, nF = 44100, 512, 2, 24
    torch.manual_seed(51)
    model = pkg.CombSub(SR, P, 256, 512, 256, n_unit=64, n_spk=2)
    model.unit2ctrl.pcmer_backward = True
    model = model.to(DEV).train()
    g = torch.Generator().manual_seed(52)
    f0 = syn.make_f0(B, nF, SR, P, seed=53)
    units, volume = torch.randn(B, nF, 64, generator=g), 0.2 * torch.rand(B, nF, 1, generator=g)
    dev = lambda t: t.to(DEV)
    signal, _, _ = model(dev(units), dev(f0), dev(volume), spk_id=dev(torch.LongTensor([[1], [2]])), infer=False,
                         noise=dev(syn.uniform_noise(B, nF * P, 54)))
    pkg.RSSLoss(256, 2048, 4)(signal, dev(syn.uniform_noise(B, nF * P, 55)) * 0.05, n_ffts=[700, 1500, 300, 1024]).backward()
    for n, p in model.unit2ctrl.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().max() > 0, n
