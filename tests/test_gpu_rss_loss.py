"""GPU: the random-scale spectral loss (csrc/rss_loss.cu through ddsp_svc_b200.loss.RSSLoss) against the reference's
autograd goldens and the float64 restatement, its exact cases, determinism, the CombSubSuperFast -> RSSLoss -> backward
chain against the oracle on CPU, and a short training loop.

Error model (as for the mel backward): the loss value (relative) and the gradient (relative RMS) against float64 stay
within RATIO = 3 times the fp32 reference's own error on the same case.  The spectra come from fp32 Bluestein
transforms instead of torch's FFT, so their round-off is of the same order but not the same; 1 / S_p and the sign term
amplify it in quiet bins, where a few bins may take the other sign than in float64 (counted for the fp32 oracle here,
and for the kernel source under emulation in tests/test_emu_rss_loss.py).  The loss
floor is at least one fp32 ulp of the loss: both sides round their result to fp32 once."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import CombSubSuperFast, FixedControls, RSSLoss, loss as pl, synthetic as syn
from tests import report, util
from tests import rss_loss_closed_form as CF
from tests.golden import make_golden_rss_loss as GR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RATIO = 3.0
SR, P, WIN, NB = 44100, 512, 2048, 1025


def _oracle_sign_flips(x_pred, x_true, n_ffts, eps=1e-7):
    """bins whose sign(log S_t - log S_p) differs between the fp32 ORACLE (torch.stft on CPU) and float64: the context
    of the error floor.  The kernels do not expose their spectra; their own count comes from the kernel source under
    host emulation (tests/test_emu_rss_loss.py::test_kernel_sign_disagreements_with_float64_are_counted)."""
    from oracle import loss as ol
    flips = 0
    for n in n_ffts:
        s32 = torch.sign(torch.log(ol.spectrogram(x_true, n, n) + eps) - torch.log(ol.spectrogram(x_pred, n, n) + eps))
        s64 = torch.sign(torch.log(ol.spectrogram(x_true.double(), n, n) + eps) -
                         torch.log(ol.spectrogram(x_pred.double(), n, n) + eps))
        flips += int((s32.double() != s64).sum())
    return flips


def gpu_loss_grad(x_pred, x_true, n_ffts):
    xp = torch.as_tensor(x_pred).to(DEV).requires_grad_(True)
    loss = RSSLoss(256, 2048, len(n_ffts))(xp, torch.as_tensor(x_true).to(DEV), n_ffts=n_ffts)
    loss.backward()
    return loss.detach().cpu().double().item(), xp.grad.cpu().numpy()


@pytest.mark.parametrize("name", list(GR.CASES))
def test_loss_and_gradient_match_float64_within_error_model(name):
    z = np.load(GR.path(name))
    n_ffts = [int(v) for v in z["n_ffts"]]
    x_true32 = z["x_true"].astype(np.float32)
    ref_loss, ref_grad, _ = CF.loss_and_grad(z["x_pred"], x_true32, n_ffts)
    floor_l = max(abs(float(z["loss"]) - ref_loss), np.spacing(np.float32(ref_loss))) / ref_loss
    floor_g = util.rms(z["grad"] - ref_grad) / util.rms(ref_grad)
    loss, grad = gpu_loss_grad(z["x_pred"], z["x_true"], n_ffts)         # fp16 x_true goes in as float16
    assert np.isfinite(grad).all() and grad.shape == z["x_pred"].shape
    el = abs(loss - ref_loss) / ref_loss
    eg = util.rms(grad - ref_grad) / util.rms(ref_grad)
    flips = _oracle_sign_flips(torch.from_numpy(z["x_pred"]), torch.from_numpy(x_true32), n_ffts)
    report.record("rss_loss/" + name, loss_err=el, loss_bound=RATIO * floor_l, grad_err=eg, grad_bound=RATIO * floor_g,
                  oracle_fp32_sign_flips=flips)
    assert el <= RATIO * floor_l, (name, el, floor_l)
    assert eg <= RATIO * floor_g, (name, eg, floor_g)


def test_equal_row_gives_exactly_zero():
    z = np.load(GR.path("rss_equal_row"))
    n_ffts = [int(v) for v in z["n_ffts"]]
    xp, xt = torch.from_numpy(z["x_pred"]).to(DEV), torch.from_numpy(z["x_true"]).to(DEV)
    assert torch.equal(xp[1], xt[1])
    _, grad = gpu_loss_grad(z["x_pred"], z["x_true"], n_ffts)
    assert not np.any(grad[1]) and np.abs(grad[0]).max() > 0
    loss, norms = pl.rss_loss_forward(xp, xt, n_ffts)
    assert torch.all(norms[:, 1, 0] == 0) and torch.all(norms[:, 0, 0] > 0)
    alone, _ = pl.rss_loss_forward(xp[1:2].contiguous(), xt[1:2].contiguous(), n_ffts)
    assert alone.item() == 0.0


def test_samples_past_the_last_frame_get_zero_gradient():
    z = np.load(GR.path("rss_ragged_t"))
    n_ffts = [int(v) for v in z["n_ffts"]]
    T = z["x_pred"].shape[1]
    end = max((T // n) * n for n in n_ffts)
    assert end < T
    _, grad = gpu_loss_grad(z["x_pred"], z["x_true"], n_ffts)
    assert not np.any(grad[:, end:]) and np.all(np.abs(grad[:, :end]).max(1) > 0)


def test_seeded_draw_matches_pinned_scales():
    z = np.load(GR.path("rss_seeded_b2_h24"))
    xp, xt = torch.from_numpy(z["x_pred"]).to(DEV), torch.from_numpy(z["x_true"]).to(DEV)
    crit = RSSLoss(256, 2048, 4)
    torch.manual_seed(1)
    a = crit(xp, xt)
    torch.manual_seed(1)
    n_ffts = torch.randint(256, 2048, (4,))
    b = crit(xp, xt, n_ffts=n_ffts)
    assert n_ffts.tolist() == z["n_ffts"].tolist()
    assert a.dim() == 0 and a.dtype == torch.float32 and a.is_cuda and torch.equal(a, b)


def test_deterministic_and_forward_under_grad_equals_no_grad():
    z = np.load(GR.path("rss_pinned_all_sizes"))
    n_ffts = [int(v) for v in z["n_ffts"]]
    l1, g1 = gpu_loss_grad(z["x_pred"], z["x_true"], n_ffts)
    l2, g2 = gpu_loss_grad(z["x_pred"], z["x_true"], n_ffts)
    assert l1 == l2 and np.array_equal(g1, g2)
    with torch.no_grad():
        l3 = RSSLoss(256, 2048, 9)(torch.from_numpy(z["x_pred"]).to(DEV), torch.from_numpy(z["x_true"]).to(DEV),
                                   n_ffts=n_ffts)
    assert l3.item() == l1


def test_argument_errors():
    x = torch.randn(2, 4000, device=DEV)
    with pytest.raises(NotImplementedError):
        RSSLoss(256, 2048, 4, overlap=0.5)
    with pytest.raises(NotImplementedError):
        RSSLoss(128, 2048, 4)
    with pytest.raises(NotImplementedError):
        RSSLoss(256, 4096, 4)
    crit = RSSLoss(256, 2048, 4)
    with pytest.raises(NotImplementedError):
        crit(x, x.clone().requires_grad_(True))
    with pytest.raises(ValueError):
        crit(x.cpu(), x.cpu())
    with pytest.raises(ValueError):
        crit(x, x[:, :3999])
    with pytest.raises(ValueError):
        crit(x[:, :300], x[:, :300], n_ffts=[512])


# ---- the combsub.yaml training step: CombSubSuperFast -> RSSLoss -> backward through both ----
# The oracle side is the port under autograd on CPU with the cotangent dL/dsignal of oracle.loss evaluated at the
# KERNEL's signal: the loss's sign term is discontinuous, and the synthesizer forward differs from the port by up to its
# gate (2e-6 abs), enough to flip sign(log S_t - log S_p) in bins where the two logs nearly agree, which changes the
# exact gradient there by 2 alpha / (B K F S_p) -- a property of the loss, not an error of either backward.
# Bound on the dense control gradient (relative RMS): the synthesizer backward's own bound
# (tests/test_gpu_superfast_backward.py) plus the loss cotangent's error, which the linear synthesizer backward carries
# into the controls: at most (RATIO + 1) x the fp32 oracle cotangent's own error against float64 on the same signal
# (RATIO for the kernel's, 1 for the oracle's).
SYNTH_BOUND = {"harmonic_magnitude": 2.5e-4, "harmonic_phase": 2.5e-4, "noise_magnitude": 1e-5, "noise_phase": 1e-5}


def chain_bound(cot, signal, target, n_ffts, scale=1.0):
    ref = CF.loss_and_grad(signal.numpy(), target.numpy(), n_ffts)[1] * scale
    floor = util.rms(cot.numpy() - ref) / util.rms(ref)
    return {k: v + (RATIO + 1) * floor for k, v in SYNTH_BOUND.items()}


SPLIT = syn.superfast_split_map(WIN)


def _rel_errs(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return {k: util.rms(got[..., i * NB:(i + 1) * NB] - ref[..., i * NB:(i + 1) * NB]) /
            util.rms(ref[..., i * NB:(i + 1) * NB]) for i, k in enumerate(SPLIT)}


def _chain_inputs(B, nF, seed):
    f0 = syn.make_f0(B, nF, SR, P, seed=seed)
    dense, _ = syn.make_ctrl(B, nF, SPLIT, seed=seed + 1)
    teacher, _ = syn.make_ctrl(B, nF, SPLIT, seed=seed + 2)
    noise = syn.normal_noise((B, nF * P), seed + 3)
    from oracle import torch_port as tp
    with torch.no_grad():
        target = tp.superfast_forward(f0, syn.split_views(teacher, SPLIT), SR, P, WIN, noise=noise)["signal"]
    return f0, dense, noise, target


def _gpu_chain_grad(f0, dense, noise, target, n_ffts):
    B, nF = dense.shape[:2]
    leaf = dense.to(DEV).requires_grad_(True)
    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=FixedControls(syn.split_views(leaf, SPLIT),
                                                                  torch.zeros(B, nF, 256, device=DEV))).to(DEV)
    signal, _, _ = model(None, f0.to(DEV), None, noise=noise.to(DEV), infer=False)
    RSSLoss(256, 2048, len(n_ffts))(signal, target.to(DEV), n_ffts=n_ffts).backward()
    return leaf.grad.cpu(), signal.detach().cpu()


def _oracle_cotangent(signal, target, n_ffts, scale=1.0):
    """dL/dsignal of oracle.loss (fp32, CPU) at ``signal``"""
    from oracle import loss as ol
    s = signal.clone().requires_grad_(True)
    (ol.rss_loss(s, target, n_ffts) * scale).backward()
    return s.grad


def _port_chain_grad(f0, dense, noise, cot):
    from oracle import torch_port as tp
    leaf = dense.clone().requires_grad_(True)
    sig = tp.superfast_forward(f0, syn.split_views(leaf, SPLIT), SR, P, WIN, noise=noise)["signal"]
    (sig * cot).sum().backward()
    return leaf.grad


@pytest.mark.parametrize("B", [2, 4])
def test_superfast_to_rss_loss_chain_matches_oracle(B):
    f0, dense, noise, target = _chain_inputs(B, 24, 30 + B)
    n_ffts = [1061, 257, 2047, 640]
    got, sig = _gpu_chain_grad(f0, dense, noise, target, n_ffts)
    cot = _oracle_cotangent(sig, target, n_ffts)
    want = _port_chain_grad(f0, dense, noise, cot)
    e = _rel_errs(got.numpy(), want.numpy())
    bound = chain_bound(cot, sig, target, n_ffts)
    report.record("rss_loss/chain_b%d" % B, **e, **{"bound_" + k: v for k, v in bound.items()})
    for k, v in e.items():
        assert v <= bound[k], (k, v, bound[k])


def test_training_batch_chain_sampled_rows_match_oracle():
    """24 x 172 hops (the 2 s crops of configs/combsub.yaml): finite gradients; two rows against the oracle on CPU.
    Every term of the loss is a mean over the batch, so a row's gradient on its own is B_sub / B times its gradient in
    the batch."""
    B, nF = 24, 172
    f0, dense, noise, target = _chain_inputs(B, nF, 50)
    n_ffts = [1800, 333, 1024, 1531]
    got, sig = _gpu_chain_grad(f0, dense, noise, target, n_ffts)
    assert torch.isfinite(got).all()
    for r in (3, 20):
        cot = _oracle_cotangent(sig[r:r + 1], target[r:r + 1], n_ffts, scale=1.0 / B)
        want = _port_chain_grad(f0[r:r + 1], dense[r:r + 1], noise[r:r + 1], cot)
        e = _rel_errs(got[r:r + 1].numpy(), want.numpy())
        bound = chain_bound(cot, sig[r:r + 1], target[r:r + 1], n_ffts, scale=1.0 / B)
        report.record("rss_loss/chain_b24_row%d" % r, **e, **{"bound_" + k: v for k, v in bound.items()})
        for k, v in e.items():
            assert v <= bound[k], (r, k, v, bound[k])


class _LinearControls(torch.nn.Module):
    """A small trainable unit2ctrl: Linear(units) -> split_to_dict (reference ddsp/unit2control.py:12-23)."""

    def __init__(self, n_in, bias):
        super().__init__()
        self.lin = torch.nn.Linear(n_in, 4 * NB)
        with torch.no_grad():
            self.lin.weight.mul_(0.1)
            self.lin.bias.copy_(bias)

    def forward(self, units, f0, phase, volume, **kw):
        return syn.split_views(self.lin(units), SPLIT), None


def test_adam_lowers_the_rss_loss_through_a_linear_unit2ctrl():
    from oracle import torch_port as tp
    B, nF, n_in = 2, 40, 16
    n_ffts = [700, 1500, 300, 1024]
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
    ref = _LinearControls(n_in, means)
    ref.load_state_dict(u2c.state_dict())

    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=u2c).to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    crit = RSSLoss(256, 2048, 4)
    f0d, ud, nd, td = f0.to(DEV), units.to(DEV), noise.to(DEV), target.to(DEV)
    losses = []
    for step in range(20):
        opt.zero_grad()
        signal, _, _ = model(ud, f0d, None, noise=nd)
        loss = crit(signal, td, n_ffts=n_ffts)
        loss.backward()
        if step == 0:                   # port on CPU, cotangent of oracle.loss at the kernel's signal (see above)
            out = tp.superfast_forward(f0, ref(units, None, None, None)[0], SR, P, WIN, noise=noise)["signal"]
            cot = _oracle_cotangent(signal.detach().cpu(), target, n_ffts)
            (out * cot).sum().backward()
            bound = chain_bound(cot, signal.detach().cpu(), target, n_ffts)["harmonic_magnitude"]
            for name in ("weight", "bias"):
                got, want = getattr(u2c.lin, name).grad.cpu(), getattr(ref.lin, name).grad
                e = util.rms(got - want) / util.rms(want)
                report.record("rss_loss/adam_first_step_" + name, err=e)
                assert e <= bound, (name, e, bound)
        opt.step()
        losses.append(loss.item())
    report.record("rss_loss/adam", first=losses[0], last=losses[-1])
    assert np.isfinite(losses).all() and losses[-1] < 0.8 * losses[0], losses


def test_prebuild_tables_builds_every_drawable_size():
    crit = RSSLoss(2000, 2048, 4)
    crit.prebuild_tables(DEV)
    idx = torch.device(DEV).index
    assert all((n, idx) in pl._tables for n in range(2000, 2048))
    t = pl._tables[(2047, idx)]
    assert t.is_cuda and t.numel() == pl._lib.lib().b2d_rss_table_floats(2047)
