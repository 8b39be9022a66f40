"""GPU: Sins trains on the kernels (training phase, infer=False).  The CUDA backward (sins_bwd.cu through
ops._SinsSynth) against the reference's autograd gradients and the oracle port, its determinism, a directional
derivative with in-kernel noise, shard invariance, the switches, the full-size shape, the sins.yaml step with RSSLoss,
a short training loop and the refusals."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import FixedControls, RSSLoss, Sins, ops, synthetic as syn
from tests import report, util
from tests import sins_grad_closed_form as cfg
from tests.golden import make_golden_sins_grad as GG
from tests.test_oracle_sins_grad import KEYS, error_model, split_grad

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P = GG.SR, GG.P
# error model (tests/test_oracle_sins_grad.error_model): relative RMS per control against float64 at the kernels' phase,
# within RATIO x the fp32 reference's own error against float64 at its phase, and not below the random-rounding floor
# of one fp32 sum of 2P products
RATIO, FLOOR = 3.0, 2.0 ** -24 * np.sqrt(2 * P)
# Where the reference side computes its own sinusoids (the port at 32 x 10 s), the all-pass bound also carries the
# relative error of the GPU forward's sinusoids against float64 (the bank's SFU sines, DESIGN §4.2), sinusoid_error().


def sinusoid_error(f0, c_amp):
    """relative RMS of the GPU oscillator bank (training phase) against float64 at the kernels' phase"""
    fph, _ = ops.phase_scan(f0.to(DEV), P, SR, infer=False)
    got = ops.sins_bank(f0.to(DEV), fph, c_amp.to(DEV), P, SR, infer=False).cpu().numpy()
    want = cfg.sinusoids(f0.numpy(), c_amp.numpy(), cfg.kernel_phase(f0.numpy(), SR, P), SR, P, reference_rounding=False)
    return util.rms(got - want) / util.rms(want)


def bounds(ref_err, e_x, ratio=RATIO):
    return {k: max(ratio * ref_err[k], FLOOR) + (e_x if k == "group_delay" else 0.0) for k in KEYS}


def model_out(name_or_split, f0, dense, noise=None, seed=None, infer=False, **kw):
    split = GG.split_map(name_or_split) if isinstance(name_or_split, str) else name_or_split
    H, Ma, Mn = split.values()
    B, nF = dense.shape[0], dense.shape[1]
    leaf = dense.detach().to(DEV).requires_grad_(True)
    model = Sins(SR, P, H, Ma, Mn, unit2ctrl=FixedControls(syn.split_views(leaf, split),
                                                           torch.zeros(B, nF, 256, device=DEV))).to(DEV)
    if seed is not None:
        torch.manual_seed(seed)
    signal, _, (harmonic, noise_out) = model(None, f0.to(DEV), None, noise=None if noise is None else noise.to(DEV),
                                             infer=infer, **kw)
    return leaf, signal, harmonic, noise_out


def model_grad(name, inp, noise="explicit", seed=None):
    leaf, sig, harm, nz = model_out(name, inp["f0"], inp["dense"], noise=inp["noise"] if noise == "explicit" else None,
                                    seed=seed)
    d = {k: (None if inp[k] is None else inp[k].to(DEV)) for k in ("cot", "cot_h", "cot_n")}
    GG.objective(sig, harm, nz, d).backward()
    return leaf.grad, sig.detach()


def gpu_sinusoids(f0, c_amp):
    """the oscillator bank output the training-phase forward stores (same kernel, same inputs)"""
    fph, _ = ops.phase_scan(f0.to(DEV), P, SR, infer=False)
    return ops.sins_bank(f0.to(DEV), fph, c_amp.to(DEV), P, SR, infer=False).cpu().numpy()


@pytest.mark.parametrize("name", list(GG.CASES))
def test_gradient_matches_reference_golden(name):
    """Each control against float64 at the kernels' phase; the all-pass gradient as the adjoint of the sinusoids this
    GPU forward produced (its SFU sines, DESIGN §4.2, are the forward's error, not the backward's)."""
    inp = GG.build_inputs(name)
    truth, ref_err = error_model(inp, np.load(GG.path(name))["grad"], name)
    truth["group_delay"] = cfg.sins_grad(
        inp["f0"].numpy(), {k: v.numpy() for k, v in inp["ctrls"].items()},
        cfg.kernel_phase(inp["f0"].numpy(), SR, P), SR, P, inp["noise"].numpy(), inp["cot"].numpy(),
        None if inp["cot_h"] is None else inp["cot_h"].numpy(), None if inp["cot_n"] is None else inp["cot_n"].numpy(),
        reference_rounding=False, sinusoids_in=gpu_sinusoids(inp["f0"], inp["ctrls"]["amplitudes"]))["group_delay"]
    grad, _ = model_grad(name, inp)
    assert torch.isfinite(grad).all()
    got = split_grad(name, grad.cpu().numpy())
    errs = {k: util.rms(got[k] - truth[k]) / util.rms(truth[k]) for k in KEYS}
    bound = bounds(ref_err, 0.0)
    report.record("sins_backward/" + name, **{k: errs[k] for k in KEYS}, **{"bound_" + k: bound[k] for k in KEYS})
    for k in KEYS:
        assert errs[k] <= bound[k], (name, k, errs[k], bound[k])


def test_forward_under_grad_is_bit_identical_to_no_grad():
    name = "sins_grad_b2_f24_h128"
    inp = GG.build_inputs(name)
    _, sig, harm, nz = model_out(name, inp["f0"], inp["dense"], seed=5)
    assert sig.requires_grad and harm.requires_grad and nz.requires_grad
    with torch.no_grad():
        _, ref, rh, rn = model_out(name, inp["f0"], inp["dense"], seed=5)
    assert torch.equal(sig, ref) and torch.equal(harm, rh) and torch.equal(nz, rn)


def test_backward_is_deterministic():
    name = "sins_grad_b2_f24_h128"
    inp = GG.build_inputs(name)
    a, _ = model_grad(name, inp, noise="kernel", seed=9)
    b, _ = model_grad(name, inp, noise="kernel", seed=9)
    assert torch.equal(a, b)
    c, _ = model_grad(name, inp)
    d, _ = model_grad(name, inp)
    assert torch.equal(c, d)


def _loss_fn(name, f0, cot, seed, utterance_offset=0):
    f0d = f0.to(DEV)
    frame_phase, _ = ops.phase_scan(f0d, P, SR, infer=False)
    cot = cot.to(DEV).double()

    def loss(dense):
        c = syn.split_views(dense, GG.split_map(name))
        sig, _, _ = ops.sins_synth(f0d, frame_phase, c["amplitudes"], c["group_delay"], c["noise_magnitude"], P, SR,
                                   seed=seed, utterance_offset=utterance_offset, infer=False)
        return (sig.double() * cot).sum()
    return loss


@pytest.mark.parametrize("key", KEYS)
def test_directional_derivative_with_in_kernel_noise(key):
    """Fourth-order central difference of L along v against <grad, v> with the in-kernel noise: the noise-control
    gradient is O(1) off unless the backward regenerates the forward's noise stream."""
    name = "sins_grad_b2_f24_h128"
    inp = GG.build_inputs(name)
    loss = _loss_fn(name, inp["f0"], inp["cot"], seed=11)
    dense = inp["dense"].to(DEV).requires_grad_(True)
    loss(dense).backward()
    v = torch.zeros_like(inp["dense"])
    views = syn.split_views(v, GG.split_map(name))
    views[key].copy_(torch.randn(views[key].shape, generator=torch.Generator().manual_seed(12)))
    v = v.to(DEV)
    eps = 1e-2
    with torch.no_grad():
        at = lambda t: loss(dense + t * eps * v).item()
        fd = (8 * (at(1) - at(-1)) - (at(2) - at(-2))) / (12 * eps)
    an = (dense.grad.double() * v.double()).sum().item()
    report.record("sins_backward/directional_" + key, fd=fd, analytic=an)
    assert abs(fd - an) <= 2e-3 * abs(an), (key, fd, an)


def test_in_kernel_noise_gradient_is_shard_invariant():
    name = "sins_grad_b2_f24_h128"
    inp = GG.build_inputs(name)
    f0, dense, cot = inp["f0"], inp["dense"], inp["cot"]
    full = dense.to(DEV).requires_grad_(True)
    _loss_fn(name, f0, cot, seed=3)(full).backward()
    part = dense[1:].to(DEV).requires_grad_(True)
    _loss_fn(name, f0[1:], cot[1:], seed=3, utterance_offset=1)(part).backward()
    assert torch.equal(full.grad[1:], part.grad)


@pytest.mark.parametrize("switch", ["overlap0", "overlap2", "fused", "spectrum"])
def test_gradient_does_not_depend_on_the_switches(switch):
    name = "sins_grad_b2_f24_h128"
    inp = GG.build_inputs(name)
    base, _ = model_grad(name, inp, noise="kernel", seed=4)
    try:
        if switch.startswith("overlap"):
            ops.set_overlap(int(switch[-1]))
        else:
            ops.set_sins_impl(switch)
        got, _ = model_grad(name, inp, noise="kernel", seed=4)
    finally:
        ops.set_overlap(1)
        ops.set_sins_impl("auto")
    assert torch.equal(base, got)


def _port_at_phase(f0, ctrls, x, noise):
    """oracle.torch_port.sins_forward's operators (the reference's ATen ops) with the phase ``x`` [B, T, 1] in cycles"""
    from oracle import torch_port as tp
    amp = tp.harmonic_amplitudes(ctrls["amplitudes"], f0, SR)
    sinus = tp.sinusoid_bank(x, amp, P)
    ir_ap = tp.impulse_response(torch.exp(1.j * torch.cumsum(np.pi * torch.tanh(ctrls["group_delay"]), dim=-1)), "none")
    nm = torch.exp(ctrls["noise_magnitude"]) / 128
    ir_n = tp.impulse_response(torch.complex(nm, torch.zeros_like(nm)), "hann")
    return tp.ltv_fir(sinus, ir_ap) + tp.ltv_fir(noise, ir_n)


def test_full_size_gradient_sampled_rows_match_port():
    """32 x 10 s: finite gradients; two sampled utterances against the oracle port's autograd gradient on CPU
    (bit-identical to the reference, tests/test_oracle_sins_grad.py).  Over 10 s the reference's fp32 cumsum phase
    and the kernels' closed-form phase differ by up to an ulp of ~2000 cycles, which sin(2 pi h x) turns into O(0.1)
    rad at h = 128: the port runs at the kernels' phase.  Bound: (RATIO + 1) x the sins.yaml golden's reference error
    (the port carries its own fp32 error, the kernels theirs), plus the forward's sinusoid error for the all-pass."""
    name = "sins_grad_b2_f24_h128"
    inp = GG.build_inputs(name)
    _, ref_err = error_model(inp, np.load(GG.path(name))["grad"], name)
    B, nF = 32, 861
    split = GG.split_map(name)
    f0 = syn.make_f0(B, nF, SR, P, unvoiced_fraction=0.03)
    dense, views = syn.make_ctrl(B, nF, split)
    noise = torch.zeros(B, nF * P)
    rows = (5, 29)
    for r in rows:
        noise[r] = syn.uniform_noise(1, nF * P, 100 + r)[0]
    cot = torch.randn(B, nF * P, generator=torch.Generator().manual_seed(77))
    leaf, sig, _, _ = model_out(split, f0, dense, noise=noise)
    (sig * cot.to(DEV)).sum().backward()
    assert torch.isfinite(leaf.grad).all()
    for r in rows:
        f0r = f0[r:r + 1]
        pl = dense[r:r + 1].clone().requires_grad_(True)
        x = torch.from_numpy(cfg.kernel_phase(f0r.numpy(), SR, P))[..., None]
        (_port_at_phase(f0r, syn.split_views(pl, split), x, noise[r:r + 1]) * cot[r:r + 1]).sum().backward()
        got = split_grad(name, leaf.grad[r:r + 1].cpu().numpy())
        want = split_grad(name, pl.grad.numpy())
        bound = bounds(ref_err, sinusoid_error(f0r, views["amplitudes"][r:r + 1]), RATIO + 1)
        for k in KEYS:
            e = util.rms(got[k] - want[k]) / util.rms(want[k])
            report.record("sins_backward/full_row%d_%s" % (r, k), err=e, bound=bound[k])
            assert e <= bound[k], (r, k, e, bound[k])


def test_sins_yaml_step_with_rss_loss_matches_oracle():
    """Sins -> RSSLoss(256, 2048, 4) -> backward at 2 x 24 frames against the port + oracle.loss under autograd at the
    kernels' phase (at the reference's phase the port's own amplitude gradient moves by 1 %).  Truth: the same port in
    float64; bound: RATIO x the fp32 port's own error (the log-spectral loss amplifies round-off in quiet bins: 1e-3
    to 3e-2 relative on this case)."""
    from oracle import loss as oloss
    name = "sins_grad_b2_f24_h128"
    inp = GG.build_inputs(name)
    target = syn.uniform_noise(2, 24 * P, 99) * 0.01
    n_ffts = [256, 777, 1500, 2047]
    crit = RSSLoss(256, 2048, 4)
    leaf, sig, _, _ = model_out(name, inp["f0"], inp["dense"], noise=inp["noise"])
    loss = crit(sig, target.to(DEV), n_ffts=n_ffts)
    loss.backward()
    x = torch.from_numpy(cfg.kernel_phase(inp["f0"].numpy(), SR, P))[..., None]

    def port(dt):
        pl = inp["dense"].to(dt).clone().requires_grad_(True)
        out = oloss.rss_loss(_port_at_phase(inp["f0"], syn.split_views(pl, GG.split_map(name)), x.to(dt),
                                            inp["noise"].to(dt)), target.to(dt), n_ffts)
        out.backward()
        return out.item(), split_grad(name, pl.grad.numpy())
    loss32, g32 = port(torch.float32)
    loss64, g64 = port(torch.float64)
    report.record("sins_backward/rss_step_loss", got=loss.item(), port=loss32, float64=loss64)
    assert abs(loss.item() - loss64) <= RATIO * max(abs(loss32 - loss64), 2.0 ** -24 * abs(loss64))
    got = split_grad(name, leaf.grad.cpu().numpy())
    for k in KEYS:
        e = util.rms(got[k] - g64[k]) / util.rms(g64[k])
        e_ref = util.rms(g32[k] - g64[k]) / util.rms(g64[k])
        report.record("sins_backward/rss_step_" + k, err=e, port_err=e_ref)
        assert e <= RATIO * e_ref, (k, e, e_ref)


class _LinearControls(torch.nn.Module):
    """A small trainable unit2ctrl: Linear(units) -> split_to_dict (reference ddsp/unit2control.py:12-23)."""

    def __init__(self, n_in, bias, split):
        super().__init__()
        self.split = split
        self.lin = torch.nn.Linear(n_in, sum(split.values()))
        with torch.no_grad():
            self.lin.weight.mul_(0.1)
            self.lin.bias.copy_(bias)

    def forward(self, units, f0, phase, volume, **kw):
        return syn.split_views(self.lin(units), self.split), None


def test_adam_trains_a_linear_unit2ctrl():
    """20 Adam steps on the kernels lower the loss, along the same curve as the same loop through the oracle port on
    CPU (the loss plateaus near 0.68x of its start for both: the all-pass phase makes the waveform MSE non-convex)."""
    from oracle import torch_port as tp
    split = syn.sins_split_map(64, 65, 65)
    B, nF, n_in = 2, 40, 16
    f0 = syn.make_f0(B, nF, SR, P, seed=21)
    units = torch.randn(B, nF, n_in, generator=torch.Generator().manual_seed(22))
    noise = syn.uniform_noise(B, nF * P, 23)
    means = torch.tensor([-2.0] * 64 + [0.0] * 65 + [-3.0] * 65)
    torch.manual_seed(25)
    teacher = _LinearControls(n_in, means + 0.5, split)
    with torch.no_grad():
        target = tp.sins_forward(f0, teacher(units, None, None, None)[0], SR, P, noise=noise, infer=False)["signal"]

    def loop(forward, u2c, steps=20):
        opt = torch.optim.Adam(u2c.parameters(), lr=1e-2)
        out = []
        for _ in range(steps):
            opt.zero_grad()
            loss = forward(u2c)
            loss.backward()
            opt.step()
            out.append(loss.item())
        return out

    torch.manual_seed(24)
    u2c = _LinearControls(n_in, means, split)
    port_u2c = _LinearControls(n_in, means, split)
    port_u2c.load_state_dict(u2c.state_dict())
    model = Sins(SR, P, 64, 65, 65, unit2ctrl=u2c).to(DEV)
    f0d, ud, nd, td = f0.to(DEV), units.to(DEV), noise.to(DEV), target.to(DEV)
    losses = loop(lambda m: ((model(ud, f0d, None, noise=nd, infer=False)[0] - td) ** 2).mean(), u2c)
    port = loop(lambda m: ((tp.sins_forward(f0, m(units, None, None, None)[0], SR, P, noise=noise,
                                            infer=False)["signal"] - target) ** 2).mean(), port_u2c)
    report.record("sins_backward/adam", first=losses[0], last=losses[-1], port_last=port[-1])
    assert np.isfinite(losses).all() and losses[-1] < 0.75 * losses[0], losses
    assert np.allclose(losses, port, rtol=2e-3, atol=0), (losses, port)


def test_refusals():
    name = "sins_grad_b1_f5_h200_ma65_mn129"
    inp = GG.build_inputs(name)
    f0 = inp["f0"].to(DEV)
    leaf = inp["dense"].to(DEV).requires_grad_(True)
    mk = lambda H, Ma, Mn, split, lf: Sins(SR, P, H, Ma, Mn, unit2ctrl=FixedControls(syn.split_views(lf, split), None)).to(DEV)
    model = mk(200, 65, 129, GG.split_map(name), leaf)
    with pytest.raises(NotImplementedError, match="infer=False"):
        model(None, f0, None)                                       # infer=True under grad
    with pytest.raises(ValueError):
        model(None, f0, None, infer=False, signal_out=torch.empty(1, 5 * P, device=DEV))
    with pytest.raises(NotImplementedError):
        model(None, f0.clone().requires_grad_(True), None, infer=False)
    big = syn.sins_split_map(16, 513, 65)                           # n_mag above 257
    lb = torch.zeros(1, 5, 16 + 513 + 65, device=DEV, requires_grad=True)
    with pytest.raises(NotImplementedError):
        mk(16, 513, 65, big, lb)(None, f0, None, infer=False)
    blk = Sins(SR, 1024, 16, 65, 65, unit2ctrl=FixedControls(syn.split_views(
        torch.zeros(1, 5, 146, device=DEV, requires_grad=True), syn.sins_split_map(16, 65, 65)), None)).to(DEV)
    with pytest.raises(NotImplementedError):                        # block size other than 512
        blk(None, f0, None, infer=False)
    with torch.no_grad():                                           # without grad all stay allowed
        out = torch.empty(1, 5 * P, device=DEV)
        sig, _, _ = model(None, f0, None, signal_out=out)
        assert sig is out
