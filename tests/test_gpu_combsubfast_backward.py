"""GPU: CombSubFast trains on the kernels in the training phase (infer=False, what the reference's DiffusionNew solver
runs).  The CUDA backward (combsubfast_bwd_kernel through ops._CombSubFastFilter) against the reference's autograd
gradients, the float64 closed form and the oracle port; its determinism, a directional derivative with in-kernel noise,
shard and chunk invariance, the full-size shape, the DiffusionNew DDSP-loss chain, a short training loop and the
refusals.

Error model.  In the training phase the kernels round the closed-form fp64 phase to fp32; the reference rounds torch's
CPU cumsum, which accumulates in fp64.  The two fp32 phases differ by an ulp on a fraction of the samples, and sinc
amplifies a phase error by sr / f0, so the comb the kernels filter is not the comb the reference filters (a CPU model
gives 1.2e-5 relative RMS at 2 x 24 frames, 2.9e-4 at 36 x 172).  The gradient of the harmonic controls is linear in
the comb, so that source difference passes straight into it.  Hence:
* the tight test compares the kernel with the float64 closed form evaluated on the kernel's OWN comb
  (ops.comb_source(..., infer=False)): TIGHT, the fp32 floor of 1.5 single-precision transforms per frame;
* against the reference (goldens) or the port, the harmonic bound of each case is measured, not fixed: twice the
  relative RMS distance between the closed form at the reference's comb and the closed form at the kernel's comb,
  plus TIGHT.  The noise side involves no comb and is held to TIGHT throughout."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import CombSubFast, FixedControls, ops, synthetic as syn
from ddsp_svc_b200 import mel as pm
from tests import combsubfast_grad_closed_form as CF
from tests import report, util
from tests.golden import make_golden_combsubfast_grad as GG

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P, NB = GG.SR, GG.P, GG.NB
SM = GG.split_map()
TIGHT = 1e-5


def split(dense):
    d = np.asarray(dense, np.float64)
    return {k: d[..., i * NB:(i + 1) * NB] for i, k in enumerate(SM)}


def rel_errs(got, ref):
    g, r = split(got), split(ref)
    return {k: util.rms(g[k] - r[k]) / util.rms(r[k]) for k in SM}


def kernel_comb(f0, initial_phase=None):
    """the comb CombSubFast(infer=False) filters, [B, T] on the device"""
    f0d = f0.to(DEV)
    fp, _ = ops.phase_scan(f0d, P, SR, None if initial_phase is None else initial_phase.to(DEV), False)
    return ops.comb_source(f0d, fp, P, SR, infer=False)


def port_comb(f0, initial_phase=None):
    from oracle import torch_port as tp
    x, f0_up = tp.wrapped_phase(f0, SR, P, initial_phase, False)
    return torch.sinc(torch.tensor(SR) * x / (f0_up + 1e-3)).squeeze(-1)


def closed_form(comb, ctrls, noise, cot):
    g = CF.combsubfast_grad(np.asarray(comb), {k: np.asarray(v) for k, v in ctrls.items()}, P, np.asarray(noise),
                            np.asarray(cot))
    return np.concatenate([g[k] for k in SM], axis=-1)


def harmonic_bounds(ctrls, noise, cot, comb_kernel, comb_ref):
    """per-control bound against a gradient computed on the reference's comb (see the module docstring)"""
    src = rel_errs(closed_form(comb_kernel, ctrls, noise, cot), closed_form(comb_ref, ctrls, noise, cot))
    return {k: (2 * src[k] + TIGHT if k.startswith("harmonic") else TIGHT) for k in SM}, src


def model_grad(f0, dense, cot, noise=None, seed=None, initial_phase=None, infer=False):
    """dense.grad of sum(signal * cot) through CombSubFast (controls = views of a leaf dense tensor)"""
    B, nF = dense.shape[0], dense.shape[1]
    leaf = dense.detach().to(DEV).requires_grad_(True)
    model = CombSubFast(SR, P, unit2ctrl=FixedControls(syn.split_views(leaf, SM),
                                                       torch.zeros(B, nF, 256, device=DEV))).to(DEV)
    if seed is not None:
        torch.manual_seed(seed)
    kw = {} if initial_phase is None else {"initial_phase": initial_phase.to(DEV)}
    signal, hidden, (s1, s2) = model(None, f0.to(DEV), None, noise=None if noise is None else noise.to(DEV),
                                     infer=infer, **kw)
    assert s1 is signal and s2 is signal and signal.requires_grad
    (signal * cot.to(DEV)).sum().backward()
    return leaf.grad, signal.detach()


@pytest.mark.parametrize("name", list(GG.CASES))
def test_gradient_matches_reference_golden_and_closed_form(name):
    inp = GG.build_inputs(name)
    gold = np.load(GG.path(name))
    grad, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], noise=inp["noise"], initial_phase=inp["initial_phase"])
    assert grad.shape == gold["grad"].shape and torch.isfinite(grad).all()
    grad = grad.cpu().numpy()
    ck = kernel_comb(inp["f0"], inp["initial_phase"]).cpu().numpy()
    ctrls = {k: v.numpy() for k, v in inp["ctrls"].items()}
    tight = rel_errs(grad, closed_form(ck, ctrls, inp["noise"], inp["cot"]))
    bound, src = harmonic_bounds(ctrls, inp["noise"], inp["cot"], ck, port_comb(inp["f0"], inp["initial_phase"]).numpy())
    e = rel_errs(grad, gold["grad"])
    report.record("combsubfast_backward/" + name, golden=e, own_comb=tight, source=src)
    for k in SM:
        assert tight[k] <= TIGHT, (name, k, tight[k])
        assert e[k] <= bound[k], (name, k, e[k], bound[k])


def test_forward_under_grad_is_bit_identical_to_no_grad():
    inp = GG.build_inputs("csfast_grad_b2_f24")
    _, sig = model_grad(inp["f0"], inp["dense"], inp["cot"], seed=5)
    model = CombSubFast(SR, P, unit2ctrl=FixedControls(syn.split_views(inp["dense"].to(DEV), SM), None)).to(DEV)
    torch.manual_seed(5)
    with torch.no_grad():
        ref, _, _ = model(None, inp["f0"].to(DEV), None, infer=False)
    assert torch.equal(sig, ref)


def test_backward_is_deterministic():
    inp = GG.build_inputs("csfast_grad_b1_f70")
    a, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], seed=9)
    b, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], seed=9)
    assert torch.equal(a, b)
    c, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], noise=inp["noise"])
    d, _ = model_grad(inp["f0"], inp["dense"], inp["cot"], noise=inp["noise"])
    assert torch.equal(c, d)


def _loss_fn(f0, cot, seed, utterance_offset=0, comb_scale=1.0):
    comb = kernel_comb(f0) * comb_scale
    cot = cot.to(DEV).double()

    def loss(dense):
        c = syn.split_views(dense, SM)
        sig = ops.combsubfast_filter(comb, c["harmonic_magnitude"], c["harmonic_phase"], c["noise_magnitude"], P,
                                     seed=seed, utterance_offset=utterance_offset)
        return (sig.double() * cot).sum()
    return loss


@pytest.mark.parametrize("side", ["harmonic", "noise"])
def test_directional_derivative_with_in_kernel_noise(side):
    """Finite difference of L along v against <grad, v> with the in-kernel noise: the backward must regenerate the
    forward's noise stream, otherwise the noise-control gradient is off by O(1).  The phase control enters as
    exp(j pi eps v), so a two-point central difference at eps = 1e-2 is itself off by ~eps^2 pi^2 v^2 / 6; the
    fourth-order stencil is accurate to < 1e-4 at the same eps.  The noise side runs without the comb: the noise part
    of L is ~600x smaller than the harmonic part, so with the comb the fp32 rounding of the signal (~2e-5 absolute
    in the difference quotient) would swamp it."""
    inp = GG.build_inputs("csfast_grad_b2_f24")
    loss = _loss_fn(inp["f0"], inp["cot"], seed=11, comb_scale=1.0 if side == "harmonic" else 0.0)
    dense = inp["dense"].to(DEV).requires_grad_(True)
    loss(dense).backward()
    g = torch.Generator().manual_seed(12)
    v = torch.zeros_like(inp["dense"])
    lo, hi = (0, 2 * NB) if side == "harmonic" else (2 * NB, 3 * NB)
    v[..., lo:hi] = torch.randn(v.shape[0], v.shape[1], hi - lo, generator=g)
    v = v.to(DEV)
    eps = 1e-2
    with torch.no_grad():
        at = lambda t: loss(dense + t * eps * v).item()
        fd = (8 * (at(1) - at(-1)) - (at(2) - at(-2))) / (12 * eps)
    an = (dense.grad.double() * v.double()).sum().item()
    report.record("combsubfast_backward/directional_" + side, fd=fd, analytic=an)
    assert abs(fd - an) <= 1e-3 * abs(an), (side, fd, an)


def test_rows_are_bit_identical_alone_and_in_a_batch():
    """Row r of a B = 32 call (4 rows per CTA) equals the same utterance computed alone (B = 1: 2 rows per CTA) with
    the same in-kernel noise stream, bit for bit; odd frame count, so frames nF-1 and nF share the last pair."""
    B, nF = 32, 41
    f0 = syn.make_f0(B, nF, SR, P, seed=51, unvoiced_fraction=0.1)
    dense, _ = syn.make_ctrl(B, nF, SM, seed=52)
    cot = torch.randn(B, nF * P, generator=torch.Generator().manual_seed(53)).to(DEV)
    comb = kernel_comb(f0)
    d = dense.to(DEV)
    c = syn.split_views(d, SM)
    full = ops.combsubfast_filter_backward(comb, c["harmonic_magnitude"], c["harmonic_phase"], c["noise_magnitude"],
                                           cot, P, seed=8)
    assert torch.isfinite(full).all()
    for r in (0, 17, 31):
        cr = syn.split_views(d[r:r + 1], SM)
        alone = ops.combsubfast_filter_backward(comb[r:r + 1], cr["harmonic_magnitude"], cr["harmonic_phase"],
                                                cr["noise_magnitude"], cot[r:r + 1], P, seed=8, utterance_offset=r)
        assert torch.equal(full[r:r + 1], alone), r


def _port_row_grad(f0, dense, noise, cot):
    from oracle import torch_port as tp
    leaf = dense.clone().requires_grad_(True)
    out = tp.combsubfast_forward(f0, syn.split_views(leaf, SM), SR, P, noise=noise, infer=False)
    (out["signal"] * cot).sum().backward()
    return leaf.grad.numpy(), out["comb"].detach().numpy()


def test_full_size_gradient_sampled_rows_match_port():
    """32 x 10 s (861 frames): finite gradients; two sampled utterances against the oracle port's autograd gradient
    on CPU (licensed bit-identical to the reference by tests/test_oracle_combsubfast_grad.py), with the source bound
    of the module docstring, and against the closed form on the kernel's own comb."""
    B, nF = 32, 861
    f0 = syn.make_f0(B, nF, SR, P, unvoiced_fraction=0.03)
    dense, _ = syn.make_ctrl(B, nF, SM)
    rows = (5, 29)
    noise = torch.zeros(B, nF * P)
    for r in rows:
        noise[r] = syn.uniform_noise(1, nF * P, 100 + r)[0]
    cot = torch.randn(B, nF * P, generator=torch.Generator().manual_seed(77))
    grad, _ = model_grad(f0, dense, cot, noise=noise)
    assert torch.isfinite(grad).all()
    ck = kernel_comb(f0).cpu().numpy()
    for r in rows:
        want, cr = _port_row_grad(f0[r:r + 1], dense[r:r + 1], noise[r:r + 1], cot[r:r + 1])
        ctrls = split(dense[r:r + 1].numpy())
        got = grad[r:r + 1].cpu().numpy()
        tight = rel_errs(got, closed_form(ck[r:r + 1], ctrls, noise[r:r + 1], cot[r:r + 1]))
        bound, src = harmonic_bounds(ctrls, noise[r:r + 1], cot[r:r + 1], ck[r:r + 1], cr)
        e = rel_errs(got, want)
        report.record("combsubfast_backward/full_row%d" % r, port=e, own_comb=tight, source=src)
        for k in SM:
            assert tight[k] <= TIGHT, (r, k, tight[k])
            assert e[k] <= bound[k], (r, k, e[k], bound[k])


def test_ddsp_loss_chain_at_the_diffusion_new_batch():
    """DiffusionNew's DDSP loss (reference diffusion/vocoder.py:246-253) at its batch, 36 x 2 s (172 frames):
    CombSubFast(infer=False) -> get_mel -> extract's transpose -> mse_loss -> backward.  Sampled rows of the control
    gradient against the oracle port + oracle.mel under autograd.  The reference's loss is evaluated at the kernel's
    signal value (the port's signal enters as kernel_signal + (s - s.detach())): the log-mel gradient divides by the
    mel value, so in quiet bands it amplifies the source difference of the two signals (1e-2 relative on the control
    gradient when each chain is differentiated at its own signal).  At the same point, the bound adds the mel chain's
    own error, 5e-4 (the bound of the same chain through CombSubSuperFast, tests/test_gpu_mel_backward.py), to the
    source bound of the module docstring evaluated on each row's dL/dsignal."""
    from oracle import mel as om
    from oracle import torch_port as tp
    B, nF = 36, 172
    f0 = syn.make_f0(B, nF, SR, P, seed=61, unvoiced_fraction=0.05)
    dense, _ = syn.make_ctrl(B, nF, SM, seed=62)
    rows = (2, 33)
    noise = torch.zeros(B, nF * P)
    for r in rows:
        noise[r] = syn.uniform_noise(1, nF * P, 300 + r)[0]
    leaf = dense.to(DEV).requires_grad_(True)
    model = CombSubFast(SR, P, unit2ctrl=FixedControls(syn.split_views(leaf, SM),
                                                       torch.zeros(B, nF, 256, device=DEV))).to(DEV)
    signal, _, _ = model(None, f0.to(DEV), None, noise=noise.to(DEV), infer=False)
    ddsp_mel = pm.STFT(SR, 128, 2048, 2048, 512, 40, 16000).get_mel(signal).transpose(1, 2)
    gt_spec = ddsp_mel.detach().cpu() + 0.3 * torch.randn(ddsp_mel.shape, generator=torch.Generator().manual_seed(63))
    torch.nn.functional.mse_loss(ddsp_mel, gt_spec.to(DEV)).backward()
    assert torch.isfinite(leaf.grad).all()
    ck = kernel_comb(f0).cpu().numpy()
    ks = signal.detach().cpu()
    n_total = ddsp_mel.numel()
    for r in rows:
        lr = dense[r:r + 1].clone().requires_grad_(True)
        out = tp.combsubfast_forward(f0[r:r + 1], syn.split_views(lr, SM), SR, P, noise=noise[r:r + 1], infer=False)
        sig = ks[r:r + 1] + (out["signal"] - out["signal"].detach())
        sig.retain_grad()
        m = om.get_mel(sig).transpose(1, 2)
        (((m - gt_spec[r:r + 1]) ** 2).sum() / n_total).backward()
        _, src = harmonic_bounds(split(dense[r:r + 1].numpy()), noise[r:r + 1], sig.grad, ck[r:r + 1],
                                 out["comb"].detach().numpy())
        e = rel_errs(leaf.grad[r:r + 1].cpu().numpy(), lr.grad.numpy())
        report.record("combsubfast_backward/chain_row%d" % r, port=e, source=src)
        for k in SM:
            bound = 5e-4 + (2 * src[k] if k.startswith("harmonic") else 0.0)
            assert e[k] <= bound, (r, k, e[k], bound)


class _LinearControls(torch.nn.Module):
    """A small trainable unit2ctrl: Linear(units) -> split_to_dict (reference ddsp/unit2control.py:12-23)."""

    def __init__(self, n_in, bias):
        super().__init__()
        self.lin = torch.nn.Linear(n_in, 3 * NB)
        with torch.no_grad():
            self.lin.weight.mul_(0.1)
            self.lin.bias.copy_(bias)

    def forward(self, units, f0, phase, volume, **kw):
        return syn.split_views(self.lin(units), SM), None


def test_adam_trains_a_linear_unit2ctrl():
    """20 Adam steps on the signal MSE against a teacher; the first step's parameter gradients against the port's
    (bound 2.5e-4 relative RMS, as for CombSubSuperFast: the source difference at 2 x 40 frames is ~1e-5)."""
    from oracle import torch_port as tp
    B, nF, n_in = 2, 40, 16
    f0 = syn.make_f0(B, nF, SR, P, seed=21)
    units = torch.randn(B, nF, n_in, generator=torch.Generator().manual_seed(22))
    noise = syn.uniform_noise(B, nF * P, 23)
    means = torch.tensor([-2.0] * NB + [0.0] * NB + [-3.0] * NB)
    torch.manual_seed(24)
    u2c = _LinearControls(n_in, means)
    torch.manual_seed(25)
    teacher = _LinearControls(n_in, means + 0.5)
    with torch.no_grad():
        target = tp.combsubfast_forward(f0, teacher(units, None, None, None)[0], SR, P, noise=noise,
                                        infer=False)["signal"]
    ref = _LinearControls(n_in, means)
    ref.load_state_dict(u2c.state_dict())
    out = tp.combsubfast_forward(f0, ref(units, None, None, None)[0], SR, P, noise=noise, infer=False)["signal"]
    ((out - target) ** 2).mean().backward()

    model = CombSubFast(SR, P, unit2ctrl=u2c).to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    f0d, ud, nd, td = f0.to(DEV), units.to(DEV), noise.to(DEV), target.to(DEV)
    losses = []
    for step in range(20):
        opt.zero_grad()
        signal, _, _ = model(ud, f0d, None, noise=nd, infer=False)
        loss = ((signal - td) ** 2).mean()
        loss.backward()
        if step == 0:
            for name in ("weight", "bias"):
                got, want = getattr(u2c.lin, name).grad.cpu(), getattr(ref.lin, name).grad
                e = util.rms(got - want) / util.rms(want)
                report.record("combsubfast_backward/adam_first_step_" + name, err=e)
                assert e <= 2.5e-4, (name, e)
        opt.step()
        losses.append(loss.item())
    report.record("combsubfast_backward/adam", first=losses[0], last=losses[-1])
    assert np.isfinite(losses).all() and losses[-1] < 0.5 * losses[0], losses


def test_refusals():
    inp = GG.build_inputs("csfast_grad_b1_f3_unvoiced")
    leaf = inp["dense"].to(DEV).requires_grad_(True)
    model = CombSubFast(SR, P, unit2ctrl=FixedControls(syn.split_views(leaf, SM), None)).to(DEV)
    f0 = inp["f0"].to(DEV)
    with pytest.raises(NotImplementedError, match="infer=False"):
        model(None, f0, None)                                              # infer=True under grad
    with pytest.raises(NotImplementedError, match="f0"):
        model(None, f0.clone().requires_grad_(True), None, infer=False)
    comb = kernel_comb(inp["f0"])
    c = syn.split_views(leaf, SM)
    with pytest.raises(NotImplementedError, match="comb"):
        ops.combsubfast_filter(comb.clone().requires_grad_(True), c["harmonic_magnitude"], c["harmonic_phase"],
                               c["noise_magnitude"], P)
    cd = syn.split_views(leaf.detach(), SM)
    args = (comb, cd["harmonic_magnitude"], cd["harmonic_phase"], cd["noise_magnitude"])
    with pytest.raises(ValueError):
        ops.combsubfast_filter_backward(*args, torch.zeros(1, 3 * P - 4, device=DEV), P)      # wrong length
    with pytest.raises(ValueError):
        ops.combsubfast_filter_backward(*args, torch.zeros(1, 3 * P), P)                      # CPU cotangent
    with torch.no_grad():                                                  # inference stays allowed
        sig, _, _ = model(None, f0, None)
        assert torch.isfinite(sig).all()
