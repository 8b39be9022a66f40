"""The CUDA backward of Unit2Control with the convolution-only decoder (csrc/unit2control_bwd.cu + library GEMMs,
ddsp_svc_b200/unit2control.py: _NaiveFunction) on the GPU:

* each kernel alone through the C ABI against a float64 torch expression of the same op at the training batch
  (24 x 172) and at 32 x 861, run twice (bit-identical);
* every parameter gradient of the whole module against the reference's own float64 gradients (tests/golden/u2c_grad_*.npz)
  in the three GEMM modes, and against the float64 oracle (oracle/unit2control.py) at the training batch;
* determinism, forward identity with the no_grad call, launch counts, refusals, the untouched PCmer path;
* end to end: CombSubSuperFast with its own Unit2Control + RSSLoss, gradients against oracle network + oracle port +
  oracle loss, then AdamW steps."""
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import _lib, ops, synthetic as syn
from ddsp_svc_b200.unit2control import Unit2Control
from oracle.unit2control import NaiveUnit2Control
from tests import report, util
from tests.golden import make_golden_u2c_grad as GG
from tests.test_emu_u2c_backward import glu_dwconv_silu_reference

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(24, 172), (32, 861)]


def _rel(got, want):
    got, want = got.detach().double(), want.detach().double()
    return util.rms((got - want).cpu()) / max(util.rms(want.cpu()), 1e-300)


def _ws(B, T, cols=4100):
    n = _lib.lib().b2d_u2c_backward_workspace_bytes(B, T, 512, cols)
    return torch.empty(n, dtype=torch.uint8, device=DEV), n


def _rand(*shape, seed, scale=1.0):
    return (scale * torch.randn(*shape, generator=torch.Generator().manual_seed(seed))).to(DEV)


def _twice(fn):
    """run a kernel call twice into fresh NaN-filled outputs: the results must be bit-identical"""
    a, b = fn(), fn()
    for x, y in zip(a, b):
        assert torch.isfinite(x).all() and torch.equal(x, y)
    return a


# ---- the kernels alone ----
@pytest.mark.parametrize("B,T", SHAPES + [(2, 20), (1, 65)])
def test_glu_dwconv_silu_backward_kernel(B, T):
    Ci, L = 512, _lib.lib()
    h, gout = _rand(B, T, 2 * Ci, seed=1), _rand(B, T, Ci, seed=2)
    w, bias = _rand(Ci, 31, seed=3, scale=0.2), _rand(Ci, seed=4, scale=0.2)
    ws, n = _ws(B, T)

    def run():
        gh, dwb = torch.full_like(h, np.nan), torch.full((Ci, 32), np.nan, device=DEV)
        _lib.check(L.b2d_u2c_glu_dwconv_silu_backward(h.data_ptr(), w.data_ptr(), bias.data_ptr(), gout.data_ptr(), gh.data_ptr(),
                                                      dwb.data_ptr(), B, T, Ci, 31, ws.data_ptr(), n, 0), "glu backward")
        return gh, dwb

    gh, dwb = _twice(run)
    want_gh, want_dwb = glu_dwconv_silu_reference(h, w, bias, gout)
    e = dict(gh=_rel(gh, want_gh), dwb=_rel(dwb, want_dwb))
    # both ends of an utterance and the tile edge (frames 63 | 64): the halo on either side
    edges = [t for t in (0, 1, 14, 15, 16, 62, 63, 64, 65, T - 16, T - 2, T - 1) if 0 <= t < T]
    e["gh_edges"] = _rel(gh[:, edges], want_gh[:, edges])
    report.record("u2c_backward/glu/%dx%d" % (B, T), **e)
    assert e["gh"] <= 2e-6 and e["gh_edges"] <= 2e-6 and e["dwb"] <= 2e-6, e


@pytest.mark.parametrize("B,T", SHAPES)
def test_layernorm_backward_kernel(B, T):
    N, L = B * T, _lib.lib()
    x, gy = _rand(N, 256, seed=5) * 2 + 0.5, _rand(N, 256, seed=6)
    gamma = 1 + _rand(256, seed=7, scale=0.2)
    ws, n = _ws(B, T)

    def run():
        gx, dgb = torch.full_like(x, np.nan), torch.full((2, 256), np.nan, device=DEV)
        _lib.check(L.b2d_u2c_layernorm_backward(x.data_ptr(), gy.data_ptr(), gamma.data_ptr(), 1e-5, N, 256, gx.data_ptr(),
                                                dgb.data_ptr(), ws.data_ptr(), n, 0), "layernorm backward")
        return gx, dgb

    gx, dgb = _twice(run)
    xd, gd, bd = x.double().requires_grad_(True), gamma.double().requires_grad_(True), torch.zeros(256, dtype=torch.float64, device=DEV, requires_grad=True)
    want = torch.autograd.grad(F.layer_norm(xd, (256,), gd, bd, 1e-5), (xd, gd, bd), gy.double())
    e = dict(gx=_rel(gx, want[0]), dgamma=_rel(dgb[0], want[1]), dbeta=_rel(dgb[1], want[2]))
    report.record("u2c_backward/layernorm/%dx%d" % (B, T), **e)
    assert max(e.values()) <= 2e-6, e


@pytest.mark.parametrize("B,T", SHAPES + [(2, 20)])
def test_groupnorm_lrelu_backward_kernel(B, T):
    L = _lib.lib()
    x, gy = _rand(B, T, 256, seed=8) * 1.5 + 0.3, _rand(B, T, 256, seed=9)
    gamma, beta = 1 + _rand(256, seed=10, scale=0.2), _rand(256, seed=11, scale=0.2)
    stats, y = torch.empty(B * 4 * 2, dtype=torch.float64, device=DEV), x.clone()
    _lib.check(L.b2d_u2c_groupnorm_lrelu(y.data_ptr(), B, T, 256, 4, gamma.data_ptr(), beta.data_ptr(), 1e-5, 0.01, stats.data_ptr(), 0),
               "groupnorm forward")
    ws, n = _ws(B, T)

    def run():
        gx, dgb = torch.full_like(x, np.nan), torch.full((2, 256), np.nan, device=DEV)
        _lib.check(L.b2d_u2c_groupnorm_lrelu_backward(x.data_ptr(), stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1e-5, 0.01,
                                                      gy.data_ptr(), B, T, 256, 4, gx.data_ptr(), dgb.data_ptr(), ws.data_ptr(), n, 0),
                   "groupnorm backward")
        return gx, dgb

    gx, dgb = _twice(run)
    xd, gd, bd = (t.double().requires_grad_(True) for t in (x, gamma, beta))
    out = F.leaky_relu(F.group_norm(xd.transpose(1, 2), 4, gd, bd, 1e-5), 0.01).transpose(1, 2)
    want = torch.autograd.grad(out, (xd, gd, bd), gy.double())
    e = dict(gx=_rel(gx, want[0]), dgamma=_rel(dgb[0], want[1]), dbeta=_rel(dgb[1], want[2]))
    report.record("u2c_backward/groupnorm/%dx%d" % (B, T), **e)
    assert max(e.values()) <= 2e-6, e


@pytest.mark.parametrize("B,T", SHAPES)
@pytest.mark.parametrize("with_aug", [True, False])
def test_embed_backward_kernel(B, T, with_aug):
    L = _lib.lib()
    gx = _rand(B * T, 256, seed=12)
    f0 = (220.0 * 2 ** (torch.rand(B, T, generator=torch.Generator().manual_seed(13)) * 2 - 1)).to(DEV)
    f0[:, 5:9] = 0.0
    phase, volume = _rand(B, T, seed=14), _rand(B, T, seed=15, scale=0.1).abs()
    aug = _rand(B, seed=16, scale=3.0) if with_aug else None
    ws, n = _ws(B, T)

    def run():
        dtable, rowsum = torch.full((7, 256), np.nan, device=DEV), torch.full((B, 256), np.nan, device=DEV)
        _lib.check(L.b2d_u2c_embed_backward(gx.data_ptr(), f0.data_ptr(), phase.data_ptr(), volume.data_ptr(),
                                            0 if aug is None else aug.data_ptr(), B, T, dtable.data_ptr(), rowsum.data_ptr(),
                                            ws.data_ptr(), n, 0), "embed backward")
        return dtable, rowsum

    dtable, rowsum = _twice(run)
    g = gx.double().reshape(B, T, 256)
    rs = g.sum(1)
    s = [(1 + f0.double() / 700).log(), phase.double() / np.pi, volume.double()]
    want = [torch.einsum("btc,bt->c", g, s[0]), rs.sum(0), torch.einsum("btc,bt->c", g, s[1]), rs.sum(0),
            torch.einsum("btc,bt->c", g, s[2]), rs.sum(0),
            (rs * (aug.double() / 5).unsqueeze(1)).sum(0) if with_aug else torch.zeros(256, dtype=torch.float64, device=DEV)]
    e = dict(rowsum=_rel(rowsum, rs), **{"row%d" % i: _rel(dtable[i], want[i]) for i in range(6 + with_aug)})
    report.record("u2c_backward/embed/%dx%d_aug%d" % (B, T, with_aug), **e)
    assert max(e.values()) <= 2e-6 and (with_aug or not dtable[6].any()), e


@pytest.mark.parametrize("B,T", SHAPES)
@pytest.mark.parametrize("cols", [256, 1024, 4100])
def test_colsum_kernel(B, T, cols):
    N, L = B * T, _lib.lib()
    g = _rand(N, cols, seed=17) + 0.25
    ws, n = _ws(B, T)

    def run():
        out = torch.full((cols,), np.nan, device=DEV)
        _lib.check(L.b2d_u2c_colsum(g.data_ptr(), N, cols, out.data_ptr(), ws.data_ptr(), n, 0), "colsum")
        return (out,)

    e = _rel(_twice(run)[0], g.double().sum(0))
    report.record("u2c_backward/colsum/%dx%d_%d" % (B, T, cols), err=e)
    assert e <= 1e-6


@pytest.mark.parametrize("B,T", SHAPES + [(2, 1)])
def test_conv3_fold_kernel(B, T):
    gcat = _rand(B, T, 768, seed=18)

    def run():
        gx = torch.full((B, T, 256), np.nan, device=DEV)
        _lib.check(_lib.lib().b2d_u2c_conv3_fold(gcat.data_ptr(), B, T, 256, gx.data_ptr(), 0), "conv3 fold")
        return (gx,)

    x = torch.zeros(B, T, 256, dtype=torch.float64, device=DEV, requires_grad=True)
    want, = torch.autograd.grad(Unit2Control._gather3(x), x, gcat.double())
    assert _rel(_twice(run)[0], want) <= 1e-7


# ---- the whole module ----
BOUND = {"3xtf32": 2e-5, "tf32": 5e-3}
# Single-pass TF32 only: the first convolution's output carries ~1e-3 of rounding, which flips the sign of GroupNorm outputs
# near zero, and a flipped LeakyReLU element changes its gradient by a factor of 100 (slope 0.01 against 1).  Everything
# behind that mask (GroupNorm parameters, first convolution) measures 1.2e-2 to 1.4e-2 on an H100 where every other tensor
# measures 2.4e-4 to 5.6e-4; the fp32 and 3xtf32 modes show no such step (stack.0.weight 4.4e-7 / 2.6e-6).
TF32_BEHIND_LRELU = {"stack.0.weight": 5e-2, "stack.0.bias": 5e-2, "stack.1.weight": 5e-2, "stack.1.bias": 5e-2}


@pytest.mark.parametrize("mode", ["fp32", "3xtf32", "tf32"])
@pytest.mark.parametrize("name", list(GG.CASES))
def test_parameter_gradients_match_the_reference(name, mode):
    """fp32 GEMMs: each tensor within 3x the fp32 reference's own error against float64 (floor 1e-6); 3xtf32: 2e-5
    (the forward measures 2.2e-6 on the controls against 4.6e-7 for fp32); tf32: 5e-3 (TF32_BEHIND_LRELU for the tensors
    behind the convolution stack's LeakyReLU).  Relative RMS over the entries the
    golden stores."""
    gold = np.load(GG.path(name))
    m = GG.build_model(name).to(DEV).train()
    m.gemm_precision = mode
    grads = GG.gradients(m, GG.build_inputs(name), torch.float32)
    assert {n for n, g in grads.items() if g is None} == set(json.loads(str(gold["none"])))
    errs, over = {}, {}
    for n, got in GG.stored(name, grads).items():
        want = gold["f64/" + n]
        errs[n] = util.rms(got.double().numpy() - want) / util.rms(want)
        bound = max(3 * float(gold["err32/" + n]), 1e-6) if mode == "fp32" else BOUND[mode]
        if mode == "tf32" and GG.CASES[name]["use_conv_stack"]:
            bound = TF32_BEHIND_LRELU.get(n, bound)
        if not errs[n] <= bound:
            over[n] = (errs[n], bound)
    report.record("u2c_backward/module/%s/%s" % (name, mode), **errs)
    assert not over, over


def test_training_batch_gradients_match_the_float64_oracle():
    """24 x 172 at the real width (768 units, 4 x 1025 controls), default GEMM mode, every entry of every gradient"""
    name = "u2c_grad_stack_spk3_aug"
    B, T = 24, 172
    m = GG.build_model(name).to(DEV).train()
    g = torch.Generator().manual_seed(40)
    inp = dict(GG.build_inputs(name))
    inp.update(units=torch.randn(B, T, 768, generator=g), f0=220.0 * 2 ** (torch.rand(B, T, 1, generator=g) * 2 - 1),
               phase=torch.rand(B, T, 1, generator=g) * 6 - 3, volume=0.2 * torch.rand(B, T, 1, generator=g),
               spk_id=torch.randint(1, 4, (B, 1), generator=g), aug_shift=torch.randn(B, 1, 1, generator=g) * 3,
               cot_dense=torch.randn(B, T, 4100, generator=g), cot_hidden=torch.randn(B, T, 256, generator=g))
    inp["f0"][:, 30:40] = 0.0
    oracle = NaiveUnit2Control(**GG.model_kwargs(name)).train()
    oracle.load_state_dict(m.state_dict())
    want = GG.gradients(oracle.to(DEV).double(), inp, torch.float64)
    got = GG.gradients(m, inp, torch.float32)
    errs = {n: _rel(got[n], w) for n, w in want.items() if w is not None}
    assert all(got[n] is None for n, w in want.items() if w is None)
    report.record("u2c_backward/module/training_batch", **errs)
    assert max(errs.values()) <= 2e-5, {n: e for n, e in errs.items() if e > 2e-5}


def _small(stack=True, **kw):
    torch.manual_seed(7)
    return Unit2Control(64, 3, GG.SMALL, use_naive_v2=True, use_conv_stack=stack, use_pitch_aug=True, **kw).to(DEV)


def _call_inputs(B=3, T=100, seed=8):
    g = torch.Generator().manual_seed(seed)
    return dict(units=torch.randn(B, T, 64, generator=g).to(DEV), f0=(100 + 300 * torch.rand(B, T, 1, generator=g)).to(DEV),
                phase=torch.randn(B, T, 1, generator=g).to(DEV), volume=torch.rand(B, T, 1, generator=g).to(DEV),
                spk_id=torch.randint(1, 4, (B, 1), generator=g).to(DEV), aug_shift=torch.randn(B, 1, 1, generator=g).to(DEV))


def test_two_backwards_from_one_forward_are_bit_identical():
    m, inp = _small(), _call_inputs()
    ctrls, hidden = m(**inp)
    dense = torch.cat(list(ctrls.values()), -1)
    params = [p for n, p in m.named_parameters() if ".norm." not in n or not n.startswith("decoder")]
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
    full = GG.gradients(m, dict(cpu, **cot), torch.float32)
    parts = [GG.gradients(m, {k: v[b:b + 1] for k, v in dict(cpu, **cot).items()}, torch.float32) for b in range(B)]
    for n, w in full.items():
        if w is not None:
            assert _rel(sum(p[n].double() for p in parts), w) <= 2e-6, n


@pytest.mark.parametrize("stack,launches", [(False, 5), (True, 6)])
def test_forward_under_grad_is_the_no_grad_forward(stack, launches):
    """same kernels: bit-identical without the convolution stack; with it the GroupNorm statistics are accumulated with
    fp64 atomics, so two forwards may differ in the last bit.  fp32 GEMMs: embed + 3 GLU stages + LayerNorm (+ GroupNorm)"""
    m, inp = _small(stack), _call_inputs()
    m.gemm_precision = "fp32"
    with torch.no_grad():
        m(**inp)                                                  # packs the weights
        n0 = ops.launches()
        c0, h0 = m(**inp)
        assert ops.launches() - n0 == launches
    n0 = ops.launches()
    c1, h1 = m(**inp)
    assert ops.launches() - n0 == launches and h1.requires_grad and all(v.requires_grad for v in c1.values())
    m.requires_grad_(False)
    c2, h2 = m(**inp)
    assert not h2.requires_grad and not any(v.requires_grad for v in c2.values())
    for a, b in ((h0, h1), (h0, h2)) + tuple((c0[k], c1[k]) for k in c0):
        assert torch.equal(a, b) if not stack else _rel(a, b) <= 1e-6
    first = next(iter(c1.values()))
    assert first.stride(1) == m.n_out                              # still views of one dense tensor


def test_inputs_are_data_and_the_pcmer_decoder_is_unchanged():
    m, inp = _small(), _call_inputs()
    for k in ("units", "f0", "phase", "volume", "aug_shift"):
        with pytest.raises(NotImplementedError):
            m(**dict(inp, **{k: inp[k].clone().requires_grad_(True)}))
    with pytest.raises(NotImplementedError):
        m(**dict(inp, spk_mix_dict={1: 0.5, 2: 0.5}))
    with torch.no_grad():
        m(**dict(inp, spk_mix_dict={1: 0.5, 2: 0.5}))              # inference keeps it
    torch.manual_seed(7)
    pc = Unit2Control(64, 3, GG.SMALL).to(DEV).train()
    c, h = pc(**{k: v for k, v in inp.items() if k != "aug_shift"})
    assert not h.requires_grad and not any(v.requires_grad for v in c.values())


# ---- end to end ----
def test_superfast_with_its_own_unit2control_trains_on_the_rss_loss():
    from oracle import loss as ol, torch_port as tp
    SR, P, WIN, B, nF = 44100, 512, 2048, 2, 40
    n_ffts = [700, 1500, 300, 1024]
    torch.manual_seed(31)
    model = pkg.CombSubSuperFast(SR, P, WIN, n_unit=768, n_spk=2, use_pitch_aug=True)
    assert isinstance(model.unit2ctrl, Unit2Control) and model.unit2ctrl.use_naive_v2
    oracle = NaiveUnit2Control(768, 2, model.unit2ctrl.output_splits, use_pitch_aug=True).train()
    oracle.load_state_dict(model.unit2ctrl.state_dict())
    model = model.to(DEV).train()
    g = torch.Generator().manual_seed(32)
    f0 = syn.make_f0(B, nF, SR, P, seed=33)
    units, volume = torch.randn(B, nF, 768, generator=g), 0.2 * torch.rand(B, nF, 1, generator=g)
    spk, aug = torch.LongTensor([[2], [1]]), torch.tensor([[[1.5]], [[-2.0]]])
    noise = syn.normal_noise((B, nF * P), 34)
    teacher, _ = syn.make_ctrl(B, nF, syn.superfast_split_map(WIN), seed=35)
    with torch.no_grad():
        target = tp.superfast_forward(f0, syn.split_views(teacher, syn.superfast_split_map(WIN)), SR, P, WIN, noise=noise)["signal"]
    cot_h = 1e-3 * torch.randn(B, nF, 256, generator=g)            # reflow / diffusion condition on hidden
    crit = pkg.RSSLoss(256, 2048, 4)
    opt = torch.optim.AdamW(model.parameters(), lr=2e-4)
    dev = lambda t: t.to(DEV)
    losses, packs = [], []
    for step in range(8):
        opt.zero_grad()
        signal, hidden, _ = model(dev(units), dev(f0), dev(volume), spk_id=dev(spk), aug_shift=dev(aug), infer=False, noise=dev(noise))
        loss = crit(signal, dev(target), n_ffts=n_ffts) + (hidden * dev(cot_h)).sum()
        loss.backward()
        packs.append(model.unit2ctrl.__dict__["_packed"][0])
        if step == 0:            # oracle network + oracle port on the CPU, cotangent of oracle.loss at the kernels' signal
            with torch.no_grad():
                _, phase = ops.superfast_scan(dev(f0), P, SR)
            s = signal.detach().cpu().requires_grad_(True)
            ol.rss_loss(s, target, n_ffts).backward()
            ctrls, hid = oracle(units, f0, phase.cpu().reshape(B, nF, 1), volume, spk_id=spk, aug_shift=aug)
            out = tp.superfast_forward(f0, ctrls, SR, P, WIN, noise=noise)["signal"]
            ((out * s.grad).sum() + (hid * cot_h).sum()).backward()
            errs = {}
            for (n, p), (_, q) in zip(model.unit2ctrl.named_parameters(), oracle.named_parameters()):
                assert (p.grad is None) == (q.grad is None), n
                if q.grad is not None:
                    idx = GG.sample_index(q.grad.numel(), 50)
                    errs[n] = _rel(p.grad.reshape(-1).cpu()[idx], q.grad.reshape(-1)[idx])
            report.record("u2c_backward/e2e_first_step", **errs)
            assert max(errs.values()) <= 2e-3, {n: e for n, e in errs.items() if e > 2e-3}
        opt.step()
        losses.append(loss.item())
    report.record("u2c_backward/e2e_adamw", first=losses[0], last=losses[-1])
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    assert len(set(packs)) == len(packs)                           # every step packed the weights the optimizer left
