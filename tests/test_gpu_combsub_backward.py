"""GPU: the old CombSub trains on the kernels (training phase, infer=False).  The CUDA backward (combsub_bwd.cu through
ops._CombSubSynth) against the reference's autograd gradients, the float64 closed form and the oracle port, its
determinism, a directional derivative with in-kernel noise, shard and switch invariance, the full-size shape, the
train.py step with RSSLoss, a short training loop and the refusals."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import CombSub, FixedControls, RSSLoss, ops, synthetic as syn
from oracle import torch_port as tp
from tests import report, util
from tests.golden import make_golden_combsub_grad as GG
from tests.test_oracle_combsub_grad import FLOOR, KEYS, RATIO, closed_form, error_model, load, split_grad

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P = GG.SR, GG.P


def gpu_comb(f0):
    """the comb the training-phase forward filters (same kernel, same inputs), [B, T] on the CPU"""
    fph, _ = ops.phase_scan(f0.to(DEV), P, SR, infer=False)
    return ops.comb_source(f0.to(DEV), fph, P, SR, infer=False).cpu().numpy()


def model_out(split, f0, dense, noise=None, seed=None, infer=False, **kw):
    Ma, Mh, Mn = split.values()
    B, nF = dense.shape[0], dense.shape[1]
    leaf = dense.detach().to(DEV).requires_grad_(True)
    model = CombSub(SR, P, Ma, Mh, Mn, unit2ctrl=FixedControls(syn.split_views(leaf, split),
                                                               torch.zeros(B, nF, 256, device=DEV))).to(DEV)
    if seed is not None:
        torch.manual_seed(seed)
    signal, _, (harmonic, noise_out) = model(None, f0.to(DEV), None, noise=None if noise is None else noise.to(DEV),
                                             infer=infer, **kw)
    return leaf, signal, harmonic, noise_out


def model_grad(name, inp, noise="explicit", seed=None):
    leaf, sig, harm, nz = model_out(GG.split_map(name), inp["f0"], inp["dense"],
                                    noise=inp["noise"] if noise == "explicit" else None, seed=seed)
    d = {k: (None if inp[k] is None else inp[k].to(DEV)) for k in ("cot", "cot_h", "cot_n")}
    GG.objective(sig, harm, nz, d).backward()
    return leaf.grad


@pytest.mark.parametrize("name", list(GG.CASES))
def test_gradient_matches_closed_form_and_reference_golden(name):
    """Against float64 at the kernels' own comb within RATIO x the fp32 reference's own error; against the golden
    within that plus twice the distance between the float64 gradients at the two combs."""
    inp, gold = load(name)
    comb = gpu_comb(inp["f0"])
    truth, tight, bound = error_model(name, inp, gold["grad"], comb)
    got = split_grad(name, model_grad(name, inp).cpu().numpy())
    ref = split_grad(name, gold["grad"])
    for k in KEYS:
        assert np.isfinite(got[k]).all()
        e = util.rms(got[k] - truth[k]) / util.rms(truth[k])
        eg = util.rms(got[k] - ref[k]) / util.rms(ref[k])
        report.record("combsub_backward/%s_%s" % (name, k), err=e, bound=tight[k], err_golden=eg, bound_golden=bound[k])
        assert e <= tight[k], (name, k, e, tight[k])
        assert eg <= bound[k], (name, k, eg, bound[k])


def test_forward_under_grad_is_bit_identical_to_no_grad():
    name = "combsub_grad_b2_f24"
    inp = GG.build_inputs(name)
    _, sig, harm, nz = model_out(GG.split_map(name), inp["f0"], inp["dense"], seed=5)
    assert sig.requires_grad and harm.requires_grad and nz.requires_grad
    with torch.no_grad():
        _, ref, rh, rn = model_out(GG.split_map(name), inp["f0"], inp["dense"], seed=5)
    assert torch.equal(sig, ref) and torch.equal(harm, rh) and torch.equal(nz, rn)


def test_backward_is_deterministic():
    name = "combsub_grad_b2_f24"
    inp = GG.build_inputs(name)
    assert torch.equal(model_grad(name, inp, noise="kernel", seed=9), model_grad(name, inp, noise="kernel", seed=9))
    assert torch.equal(model_grad(name, inp), model_grad(name, inp))


def _loss_fn(name, f0, cot, seed, utterance_offset=0):
    f0d = f0.to(DEV)
    frame_phase, _ = ops.phase_scan(f0d, P, SR, infer=False)
    cot = cot.to(DEV).double()

    def loss(dense):
        c = syn.split_views(dense, GG.split_map(name))
        sig, _, _ = ops.combsub_synth(f0d, frame_phase, c["group_delay"], c["harmonic_magnitude"],
                                      c["noise_magnitude"], P, SR, seed=seed, utterance_offset=utterance_offset,
                                      infer=False)
        return (sig.double() * cot).sum()
    return loss


@pytest.mark.parametrize("key", KEYS)
def test_directional_derivative_with_in_kernel_noise(key):
    """Fourth-order central difference of L along v against <grad, v> with the in-kernel noise: the noise-control
    gradient is O(1) off unless the backward regenerates the forward's noise stream.  eps = 2e-3: along the all-pass
    controls the cumulative phase makes L strongly curved (at eps = 1e-2 the float64 port's own difference quotient is
    0.7 % off its exact derivative, at 3e-3 8e-5)."""
    name = "combsub_grad_b2_f24"
    inp = GG.build_inputs(name)
    loss = _loss_fn(name, inp["f0"], inp["cot"], seed=11)
    dense = inp["dense"].to(DEV).requires_grad_(True)
    loss(dense).backward()
    v = torch.zeros_like(inp["dense"])
    views = syn.split_views(v, GG.split_map(name))
    views[key].copy_(torch.randn(views[key].shape, generator=torch.Generator().manual_seed(12)))
    v = v.to(DEV)
    eps = 2e-3
    with torch.no_grad():
        at = lambda t: loss(dense + t * eps * v).item()
        fd = (8 * (at(1) - at(-1)) - (at(2) - at(-2))) / (12 * eps)
    an = (dense.grad.double() * v.double()).sum().item()
    report.record("combsub_backward/directional_" + key, fd=fd, analytic=an)
    assert abs(fd - an) <= 2e-3 * abs(an), (key, fd, an)


def test_in_kernel_noise_gradient_is_shard_invariant():
    name = "combsub_grad_b2_f24"
    inp = GG.build_inputs(name)
    f0, dense, cot = inp["f0"], inp["dense"], inp["cot"]
    full = dense.to(DEV).requires_grad_(True)
    _loss_fn(name, f0, cot, seed=3)(full).backward()
    part = dense[1:].to(DEV).requires_grad_(True)
    _loss_fn(name, f0[1:], cot[1:], seed=3, utterance_offset=1)(part).backward()
    assert torch.equal(full.grad[1:], part.grad)


@pytest.mark.parametrize("mode", [0, 2, -2])
def test_gradient_does_not_depend_on_the_overlap_mode(mode):
    name = "combsub_grad_b2_f24"
    inp = GG.build_inputs(name)
    base = model_grad(name, inp, noise="kernel", seed=4)
    try:
        ops.set_overlap(mode)
        got = model_grad(name, inp, noise="kernel", seed=4)
    finally:
        ops.set_overlap(1)
    assert torch.equal(base, got)


@pytest.mark.parametrize("impl", ["cuda"])
def test_gradient_across_fir_implementations_within_round_off(impl):
    """the forward's FIR kernel changes the stored all-passed comb in its last bits, nothing else"""
    name = "combsub_grad_b2_f24"
    inp = GG.build_inputs(name)
    base = split_grad(name, model_grad(name, inp).cpu().numpy())
    try:
        ops.set_fir_impl(impl)
        got = split_grad(name, model_grad(name, inp).cpu().numpy())
    finally:
        ops.set_fir_impl("auto")
    for k in KEYS:
        e = util.rms(got[k] - base[k]) / util.rms(base[k])
        report.record("combsub_backward/fir_%s_%s" % (impl, k), err=e)
        assert e <= 1e-5, (impl, k, e)


def _port_at_comb(f0, ctrls, comb, noise):
    """oracle.torch_port.combsub_forward's operators (the reference's ATen ops) on the comb ``comb`` [B, T]"""
    gd = np.pi * torch.tanh(ctrls["group_delay"])
    src = torch.exp(ctrls["harmonic_magnitude"])
    nm = torch.exp(ctrls["noise_magnitude"]) / 128
    allp = tp.ltv_fir(comb, tp.impulse_response(torch.exp(1.j * torch.cumsum(gd, dim=-1)), "none"))
    ir_h = tp.impulse_response(torch.complex(src, torch.zeros_like(src)), "dynamic",
                               1.5 * torch.tensor(SR) / (f0.to(comb.dtype) + 1e-3))
    ir_n = tp.impulse_response(torch.complex(nm, torch.zeros_like(nm)), "hann")
    return tp.ltv_fir(allp, ir_h) + tp.ltv_fir(noise, ir_n)


def test_full_size_gradient_sampled_rows_match_port():
    """32 x 10 s: finite gradients; two sampled utterances against the oracle port's autograd gradient on CPU at the
    kernels' comb (bit-identical to the reference on the reference's comb, tests/test_oracle_combsub_grad.py).  Bound:
    (RATIO + 1) x the b2_f24 golden's reference error (the port carries its own fp32 error, the kernels theirs)."""
    name = "combsub_grad_b2_f24"
    inp, gold = load(name)
    at_ref = closed_form(inp, tp.combsub_forward(inp["f0"], inp["ctrls"], SR, P, noise=inp["noise"],
                                                 infer=False)["comb"].numpy())
    ref_err = {k: util.rms(split_grad(name, gold["grad"])[k] - at_ref[k]) / util.rms(at_ref[k]) for k in KEYS}
    B, nF = 32, 861
    split = GG.split_map(name)
    f0 = syn.make_f0(B, nF, SR, P, unvoiced_fraction=0.03)
    dense, _ = syn.make_ctrl(B, nF, split)
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
        comb = torch.from_numpy(gpu_comb(f0r))
        (_port_at_comb(f0r, syn.split_views(pl, split), comb, noise[r:r + 1]) * cot[r:r + 1]).sum().backward()
        got = split_grad(name, leaf.grad[r:r + 1].cpu().numpy())
        want = split_grad(name, pl.grad.numpy())
        for k in KEYS:
            e = util.rms(got[k] - want[k]) / util.rms(want[k])
            bound = max((RATIO + 1) * ref_err[k], FLOOR[k])
            report.record("combsub_backward/full_row%d_%s" % (r, k), err=e, bound=bound)
            assert e <= bound, (r, k, e, bound)


def test_train_step_with_rss_loss_matches_oracle():
    """CombSub -> RSSLoss(256, 2048, 4) -> backward at 2 x 24 frames against the port + oracle.loss under autograd at
    the kernels' comb.  Truth: the same port in float64; bound: RATIO x the fp32 port's own error (the log-spectral
    loss amplifies round-off in quiet bins)."""
    from oracle import loss as oloss
    name = "combsub_grad_b2_f24"
    inp = GG.build_inputs(name)
    target = syn.uniform_noise(2, 24 * P, 99) * 0.01
    n_ffts = [256, 777, 1500, 2047]
    crit = RSSLoss(256, 2048, 4)
    leaf, sig, _, _ = model_out(GG.split_map(name), inp["f0"], inp["dense"], noise=inp["noise"])
    loss = crit(sig, target.to(DEV), n_ffts=n_ffts)
    loss.backward()
    comb = torch.from_numpy(gpu_comb(inp["f0"]))

    def port(dt):
        pl = inp["dense"].to(dt).clone().requires_grad_(True)
        out = oloss.rss_loss(_port_at_comb(inp["f0"], syn.split_views(pl, GG.split_map(name)), comb.to(dt),
                                           inp["noise"].to(dt)), target.to(dt), n_ffts)
        out.backward()
        return out.item(), split_grad(name, pl.grad.numpy())
    loss32, g32 = port(torch.float32)
    loss64, g64 = port(torch.float64)
    report.record("combsub_backward/rss_step_loss", got=loss.item(), port=loss32, float64=loss64)
    # the loss also carries the GPU forward's own fp32 error (FFT-domain FIRs): not below one fp32 sum of 2P products
    assert abs(loss.item() - loss64) <= RATIO * max(abs(loss32 - loss64), 2.0 ** -24 * np.sqrt(2 * P) * abs(loss64))
    got = split_grad(name, leaf.grad.cpu().numpy())
    for k in KEYS:
        e = util.rms(got[k] - g64[k]) / util.rms(g64[k])
        e_ref = util.rms(g32[k] - g64[k]) / util.rms(g64[k])
        report.record("combsub_backward/rss_step_" + k, err=e, port_err=e_ref)
        assert e <= max(RATIO * e_ref, FLOOR[k]), (k, e, e_ref)


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
    """20 Adam steps on the kernels lower the waveform MSE against a teacher's output (by 21 % on an H100)."""
    split = syn.combsub_split_map(65, 129, 65)
    B, nF, n_in = 2, 40, 16
    f0 = syn.make_f0(B, nF, SR, P, seed=21)
    units = torch.randn(B, nF, n_in, generator=torch.Generator().manual_seed(22))
    noise = syn.uniform_noise(B, nF * P, 23)
    means = torch.tensor([0.0] * 65 + [-2.0] * 129 + [-3.0] * 65)
    torch.manual_seed(25)
    teacher = _LinearControls(n_in, means + 0.5, split)
    with torch.no_grad():
        target = tp.combsub_forward(f0, teacher(units, None, None, None)[0], SR, P, noise=noise,
                                    infer=False)["signal"]
    torch.manual_seed(24)
    u2c = _LinearControls(n_in, means, split)
    model = CombSub(SR, P, 65, 129, 65, unit2ctrl=u2c).to(DEV)
    f0d, ud, nd, td = f0.to(DEV), units.to(DEV), noise.to(DEV), target.to(DEV)
    opt = torch.optim.Adam(u2c.parameters(), lr=1e-2)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        loss = ((model(ud, f0d, None, noise=nd, infer=False)[0] - td) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    report.record("combsub_backward/adam", first=losses[0], last=losses[-1])
    assert np.isfinite(losses).all() and losses[-1] < 0.85 * losses[0], losses


def test_refusals():
    name = "combsub_grad_b1_f5_ma65_mh129_mn33"
    inp = GG.build_inputs(name)
    f0 = inp["f0"].to(DEV)
    leaf = inp["dense"].to(DEV).requires_grad_(True)
    mk = lambda block, Ma, Mh, Mn, lf: CombSub(SR, block, Ma, Mh, Mn, unit2ctrl=FixedControls(
        syn.split_views(lf, syn.combsub_split_map(Ma, Mh, Mn)), None)).to(DEV)
    model = mk(P, 65, 129, 33, leaf)
    with pytest.raises(NotImplementedError, match="infer=False"):
        model(None, f0, None)                                       # infer=True under grad
    with pytest.raises(ValueError):
        model(None, f0, None, infer=False, signal_out=torch.empty(1, 5 * P, device=DEV))
    with pytest.raises(NotImplementedError):
        model(None, f0.clone().requires_grad_(True), None, infer=False)
    lb = torch.zeros(1, 5, 65 + 514 + 33, device=DEV, requires_grad=True)
    with pytest.raises(NotImplementedError, match="n_mag"):         # n_mag above 513
        mk(P, 65, 514, 33, lb)(None, f0, None, infer=False)
    with pytest.raises(NotImplementedError, match="block size"):    # block size other than 512
        mk(1024, 65, 129, 33, leaf)(None, f0, None, infer=False)
    with torch.no_grad():                                           # without grad all stay allowed
        out = torch.empty(1, 5 * P, device=DEV)
        sig, _, _ = model(None, f0, None, signal_out=out)
        assert sig is out
