"""GPU: CombSubSuperFast trains on the kernels.  The CUDA backward (superfast_bwd_kernel through
ops._SuperFastSynth) against the reference's autograd gradients and the oracle port, its determinism, a directional
derivative with in-kernel noise, shard invariance, the full-size shape and a short training loop."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import CombSub, CombSubFast, CombSubSuperFast, FixedControls, Sins, ops, synthetic as syn
from tests import report, util
from tests.golden import make_golden_superfast_grad as GG

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P, WIN, NB = GG.SR, GG.P, GG.WIN, GG.WIN // 2 + 1
# relative RMS per control: the harmonic bound is the forward's GATE_RMS (2e-6 abs) relative to the signal RMS (the
# GPU comb uses the SFU sine); the noise side has no comb and sits near the fp32 floor
BOUND = {"harmonic_magnitude": 2.5e-4, "harmonic_phase": 2.5e-4, "noise_magnitude": 1e-5, "noise_phase": 1e-5}


def rel_errs(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return {k: util.rms(got[..., i * NB:(i + 1) * NB] - ref[..., i * NB:(i + 1) * NB]) /
            util.rms(ref[..., i * NB:(i + 1) * NB]) for i, k in enumerate(GG.split_map())}


def model_grad(f0, dense, cot, noise=None, seed=None, **kw):
    """dense.grad of sum(signal * cot) through CombSubSuperFast (controls = views of a leaf dense tensor)"""
    B, nF = dense.shape[0], dense.shape[1]
    leaf = dense.detach().to(DEV).requires_grad_(True)
    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=FixedControls(syn.split_views(leaf, GG.split_map()),
                                                                  torch.zeros(B, nF, 256, device=DEV))).to(DEV)
    if seed is not None:
        torch.manual_seed(seed)
    signal, hidden, (s1, s2) = model(None, f0.to(DEV), None, noise=None if noise is None else noise.to(DEV), **kw)
    assert s1 is signal and s2 is signal and signal.requires_grad
    (signal * cot.to(DEV)).sum().backward()
    return leaf.grad, signal.detach()


@pytest.mark.parametrize("name", list(GG.CASES))
def test_gradient_matches_reference_golden(name):
    inp = GG.build_inputs(name)
    gold = np.load(GG.path(name))
    grad, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], noise=inp["noise"])
    assert grad.shape == gold["grad"].shape and torch.isfinite(grad).all()
    e = rel_errs(grad.cpu().numpy(), gold["grad"])
    report.record("superfast_backward/" + name, **e)
    for k, v in e.items():
        assert v <= BOUND[k], (name, k, v)


def test_forward_under_grad_is_bit_identical_to_no_grad():
    inp = GG.build_inputs("superfast_grad_b2_f24")
    _, sig = model_grad(inp["f0"], inp["dense"], inp["cot"], seed=5)
    dc = syn.split_views(inp["dense"].to(DEV), GG.split_map())
    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=FixedControls(dc, None)).to(DEV)
    torch.manual_seed(5)
    with torch.no_grad():
        ref, _, _ = model(None, inp["f0"].to(DEV), None)
    assert torch.equal(sig, ref)


def test_backward_is_deterministic():
    inp = GG.build_inputs("superfast_grad_b1_f48")
    a, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], seed=9)
    b, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], seed=9)
    assert torch.equal(a, b)
    c, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], noise=inp["noise"])
    d, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], noise=inp["noise"])
    assert torch.equal(c, d)


def _loss_fn(f0, cot, seed, utterance_offset=0):
    ws, _ = ops.superfast_scan(f0.to(DEV), P, SR)
    cot = cot.to(DEV).double()

    def loss(dense):
        c = syn.split_views(dense, GG.split_map())
        sig = ops.superfast_synth(ws, c["harmonic_magnitude"], c["harmonic_phase"], c["noise_magnitude"],
                                  c["noise_phase"], P, WIN, seed=seed, utterance_offset=utterance_offset)
        return (sig.double() * cot).sum()
    return loss


@pytest.mark.parametrize("side", ["harmonic", "noise"])
def test_directional_derivative_with_in_kernel_noise(side):
    """Finite difference of L along v against <grad, v> with the in-kernel noise: the backward must regenerate the
    forward's noise stream, otherwise the noise-control gradient is off by O(1).  The phase controls enter as
    exp(j pi eps v), so a two-point central difference at eps = 1e-2 is itself off by ~eps^2 pi^2 v^2 / 6 (1e-3 to
    2e-2 relative in float64 on these inputs); the fourth-order stencil is accurate to < 1e-4 at the same eps."""
    inp = GG.build_inputs("superfast_grad_b2_f24")
    loss = _loss_fn(inp["f0"], inp["cot"], seed=11)
    dense = inp["dense"].to(DEV).requires_grad_(True)
    loss(dense).backward()
    g = torch.Generator().manual_seed(12)
    v = torch.zeros_like(inp["dense"])
    lo = 0 if side == "harmonic" else 2 * NB
    v[..., lo:lo + 2 * NB] = torch.randn(v.shape[0], v.shape[1], 2 * NB, generator=g)
    v = v.to(DEV)
    eps = 1e-2
    with torch.no_grad():
        at = lambda t: loss(dense + t * eps * v).item()
        fd = (8 * (at(1) - at(-1)) - (at(2) - at(-2))) / (12 * eps)
    an = (dense.grad.double() * v.double()).sum().item()
    report.record("superfast_backward/directional_" + side, fd=fd, analytic=an)
    assert abs(fd - an) <= 1e-3 * abs(an), (side, fd, an)


def test_in_kernel_noise_gradient_is_shard_invariant():
    inp = GG.build_inputs("superfast_grad_b2_f24")
    f0, dense, cot = inp["f0"], inp["dense"], inp["cot"]
    full = dense.to(DEV).requires_grad_(True)
    _loss_fn(f0, cot, seed=3)(full).backward()
    part = dense[1:].to(DEV).requires_grad_(True)
    _loss_fn(f0[1:], cot[1:], seed=3, utterance_offset=1)(part).backward()
    assert torch.equal(full.grad[1:], part.grad)


def test_full_size_gradient_sampled_rows_match_port():
    """BASELINE config 3 shape (B=32 x 10 s): finite gradients; two sampled utterances against the oracle port's
    autograd gradient on CPU (licensed bit-identical to the reference by tests/test_oracle_superfast_grad.py)."""
    from oracle import torch_port as tp
    B, nF = 32, 861
    f0 = syn.make_f0(B, nF, SR, P, unvoiced_fraction=0.03)
    dense, _ = syn.make_ctrl(B, nF, GG.split_map())
    rows = (5, 29)
    noise = torch.zeros(B, nF * P)
    for r in rows:
        noise[r] = syn.normal_noise((1, nF * P), 100 + r)[0]
    cot = torch.randn(B, nF * P, generator=torch.Generator().manual_seed(77))
    grad, _ = model_grad(f0, dense, cot, noise=noise)
    assert torch.isfinite(grad).all()
    for r in rows:
        leaf = dense[r:r + 1].clone().requires_grad_(True)
        out = tp.superfast_forward(f0[r:r + 1], syn.split_views(leaf, GG.split_map()), SR, P, WIN, noise=noise[r:r + 1])
        (out["signal"] * cot[r:r + 1]).sum().backward()
        e = rel_errs(grad[r:r + 1].cpu().numpy(), leaf.grad.numpy())
        report.record("superfast_backward/full_row%d" % r, **e)
        for k, v in e.items():
            assert v <= BOUND[k], (r, k, v)


class _LinearControls(torch.nn.Module):
    """A small trainable unit2ctrl: Linear(units) -> split_to_dict (reference ddsp/unit2control.py:12-23)."""

    def __init__(self, n_in, bias):
        super().__init__()
        self.lin = torch.nn.Linear(n_in, 4 * NB)
        with torch.no_grad():
            self.lin.weight.mul_(0.1)
            self.lin.bias.copy_(bias)

    def forward(self, units, f0, phase, volume, **kw):
        return syn.split_views(self.lin(units), GG.split_map()), None


def test_adam_trains_a_linear_unit2ctrl():
    from oracle import torch_port as tp
    B, nF, n_in = 2, 40, 16
    f0 = syn.make_f0(B, nF, SR, P, seed=21)
    units = torch.randn(B, nF, n_in, generator=torch.Generator().manual_seed(22))
    noise = syn.normal_noise((B, nF * P), 23)
    means = torch.tensor([-2.0] * NB + [0.0] * NB + [-3.0] * NB + [0.0] * NB)
    torch.manual_seed(24)
    u2c = _LinearControls(n_in, means)
    torch.manual_seed(25)
    teacher = _LinearControls(n_in, means + 0.5)
    with torch.no_grad():
        target = tp.superfast_forward(f0, teacher(units, None, None, None)[0], SR, P, WIN, noise=noise)["signal"]
    # first-step parameter gradients of the same loss through the port on CPU
    ref = _LinearControls(n_in, means)
    ref.load_state_dict(u2c.state_dict())
    out = tp.superfast_forward(f0, ref(units, None, None, None)[0], SR, P, WIN, noise=noise)["signal"]
    ((out - target) ** 2).mean().backward()

    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=u2c).to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    f0d, ud, nd, td = f0.to(DEV), units.to(DEV), noise.to(DEV), target.to(DEV)
    losses = []
    for step in range(20):
        opt.zero_grad()
        signal, _, _ = model(ud, f0d, None, noise=nd)
        loss = ((signal - td) ** 2).mean()
        loss.backward()
        if step == 0:
            for name in ("weight", "bias"):
                got, want = getattr(u2c.lin, name).grad.cpu(), getattr(ref.lin, name).grad
                e = util.rms(got - want) / util.rms(want)
                report.record("superfast_backward/adam_first_step_" + name, err=e)
                assert e <= 2.5e-4, (name, e)
        opt.step()
        losses.append(loss.item())
    report.record("superfast_backward/adam", first=losses[0], last=losses[-1])
    assert np.isfinite(losses).all() and losses[-1] < 0.5 * losses[0], losses


def test_other_synthesizers_still_refuse_grad():
    f0 = syn.make_f0(1, 4, SR, P).to(DEV)
    req = lambda n: torch.zeros(1, 4, n, device=DEV, requires_grad=True)
    cases = [(Sins(SR, P, 8, 16, 16, unit2ctrl=FixedControls({"amplitudes": req(8), "group_delay": req(16),
                                                               "noise_magnitude": req(16)}, None)), {}),
             (CombSub(SR, P, 16, 16, 16, unit2ctrl=FixedControls({"group_delay": req(16), "harmonic_magnitude": req(16),
                                                                   "noise_magnitude": req(16)}, None)), {}),
             (CombSubFast(SR, P, unit2ctrl=FixedControls({"harmonic_magnitude": req(513), "harmonic_phase": req(513),
                                                          "noise_magnitude": req(513)}, None)), {})]
    for m, kw in cases:
        with pytest.raises(NotImplementedError):
            m.to(DEV)(None, f0, None, **kw)


def test_superfast_refuses_signal_out_and_f0_grad_under_grad():
    inp = GG.build_inputs("superfast_grad_b1_f5")
    leaf = inp["dense"].to(DEV).requires_grad_(True)
    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=FixedControls(syn.split_views(leaf, GG.split_map()), None)).to(DEV)
    f0 = inp["f0"].to(DEV)
    with pytest.raises(ValueError):
        model(None, f0, None, signal_out=torch.empty(1, 5 * P, device=DEV))
    with pytest.raises(NotImplementedError):
        model(None, f0.clone().requires_grad_(True), None)
    with torch.no_grad():      # without grad both stay allowed
        out = torch.empty(1, 5 * P, device=DEV)
        sig, _, _ = model(None, f0, None, signal_out=out)
        assert sig is out
