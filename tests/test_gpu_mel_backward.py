"""GPU: the mel front end's CUDA backward (mel_bwd_kernel through mel.STFT.get_mel's autograd Function), so the DDSP
loss of the reflow / diffusion models trains CombSubSuperFast on the kernels.

Error model.  Every implementation here computes the same fp32 algorithm class: 2048-point FFTs, magnitudes, a sparse
projection M = basis @ mag and gM = g / M.  The FFT's round-off is relative to the frame's spectral norm, not to each
bin, so in a quiet mel band (M far below the frame's loudest bands) the relative error of M, and with it of g / M, is
amplified by roughly (frame norm) / M.  A fixed absolute or relative bound would therefore depend on the signal.  The
bound used instead is relative to the fp32 reference itself: on each case the kernel's relative RMS error against the
float64 ground truth (tests/mel_grad_closed_form.py, which the CPU tests pin to float64 autograd of the reference's
operators and to the reference's own fp32 gradients) must be at most RATIO times the error of the reference's fp32
autograd gradient (the goldens) against the same float64 truth.  The emulated kernel source sits at 1.0-1.6x."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import CombSubSuperFast, FixedControls, synthetic as syn
from ddsp_svc_b200 import mel as pm
from oracle import mel as om
from tests import mel_grad_closed_form as CF
from tests import report, util
from tests.golden import make_golden_mel_grad as GG

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P, WIN, NB = 44100, 512, 2048, 1025
RATIO = 3.0
SM = syn.superfast_split_map(WIN)


def _stft(hop=512):
    return pm.STFT(SR, 128, 2048, 2048, hop, 40, 16000)


def kernel_grad(y, hop, cot):
    yd = torch.as_tensor(y).to(DEV).requires_grad_(True)
    mel = _stft(hop).get_mel(yd)
    assert mel.requires_grad
    (mel * torch.as_tensor(cot).to(DEV)).sum().backward()
    return yd.grad.cpu().numpy(), mel.detach()


@pytest.mark.parametrize("name", list(GG.CASES))
def test_gradient_against_golden_and_float64(name):
    z = np.load(GG.path(name))
    hop = int(z["hop"])
    got, mel = kernel_grad(z["y"], hop, z["cot"])
    assert np.isfinite(got).all()
    truth = CF.mel_grad(z["y"], hop, z["cot"])
    floor = util.rms(z["grad"] - truth) / util.rms(truth)
    e64 = util.rms(got - truth) / util.rms(truth)
    egold = util.rms(got - z["grad"]) / util.rms(truth)
    report.record("mel_backward/" + name, err_vs_f64=e64, ref_err_vs_f64=floor, ratio=e64 / floor, err_vs_golden=egold,
                  bound=RATIO * floor)
    assert e64 <= RATIO * floor, (name, e64, floor)
    assert egold <= (RATIO + 1) * floor, (name, egold, floor)


def test_clamp_consistency():
    """A cotangent only on entries whose float64 pre-log value is under clip/2 gives exactly zero; one on entries above
    2 clip gives a non-zero gradient.  (Selecting by out == log(clip) would also catch values a few ulps above the clip
    that logf rounds to the same float, where the clamp is inactive.)"""
    z = np.load(GG.path("mel_grad_b1_f172_silence"))
    M = CF.forward(z["y"], 512)[2]
    rnd = np.random.default_rng(3).standard_normal(M.shape).astype(np.float32)
    below = np.where(M < 0.5 * CF.CLIP, rnd, 0).astype(np.float32)
    above = np.where(M > 2.0 * CF.CLIP, rnd, 0).astype(np.float32)
    assert np.count_nonzero(below) > 1000 and np.count_nonzero(above) > 1000
    g0, _ = kernel_grad(z["y"], 512, below)
    assert np.count_nonzero(g0) == 0
    g1, _ = kernel_grad(z["y"], 512, above)
    report.record("mel_backward/clamp", below_entries=int(np.count_nonzero(below)), nonzero_from_below=0,
                  nonzero_from_above=int(np.count_nonzero(g1)))
    assert np.isfinite(g1).all() and np.count_nonzero(g1) > 0.5 * g1.size


def test_forward_bits_determinism_and_gradient_layout():
    B, T = 3, 172 * 512 + 301
    y = 0.1 * torch.randn(B, T, generator=torch.Generator().manual_seed(5)).to(DEV)
    st = _stft()
    with torch.no_grad():
        ref = st.get_mel(y)
    yg = y.clone().requires_grad_(True)
    out = st.get_mel(yg)
    assert out.requires_grad and torch.equal(out.detach(), ref)
    cot = torch.randn(ref.shape, generator=torch.Generator().manual_seed(6)).to(DEV)
    a = st.get_mel_backward(y, cot)
    assert torch.equal(a, st.get_mel_backward(y, cot))
    cot_t = cot.transpose(1, 2).contiguous()                  # extract's [B, F, n_mels] layout, seen transposed
    assert torch.equal(a, st.get_mel_backward(y, cot_t.transpose(1, 2)))
    (out.transpose(1, 2) * cot_t).sum().backward()            # what autograd hands get_mel after extract's transpose
    assert torch.equal(yg.grad, a)


def test_rejected_arguments_raise_under_grad_too():
    st = _stft()
    y = torch.randn(1, 8192, requires_grad=True)
    with pytest.raises(ValueError):
        st.get_mel(y)                                          # CPU tensor: no fallback
    yd = y.detach().to(DEV).requires_grad_(True)
    with pytest.raises(NotImplementedError):
        st.get_mel(yd, keyshift=2)
    with pytest.raises(NotImplementedError):
        st.get_mel(yd, speed=1.5)
    with pytest.raises(NotImplementedError):
        pm.STFT(22050, 80, 1024, 1024, 256, 20, 11025).get_mel(yd)
    with pytest.raises(ValueError):
        st.get_mel_backward(yd, torch.zeros(1, 128, 16))       # CPU cotangent
    with pytest.raises(ValueError):
        st.get_mel_backward(yd, torch.zeros(1, 128, 15, device=DEV))


def test_ddsp_loss_chain_at_the_reflow_batch():
    """CombSubSuperFast -> get_mel -> extract's transpose -> mse + a linear term, at configs/reflow.yaml's batch
    (48 x 2 s, 172 frames): sampled rows of the control gradient against the oracle port + oracle.mel under autograd.
    The bound is twice the synthesizer backward's harmonic bound (2.5e-4, tests/test_gpu_superfast_backward.py), to
    cover the mel chain's own error on top of it: 5e-4 relative RMS per control."""
    from oracle import torch_port as tp
    B, nF = 48, 172
    f0 = syn.make_f0(B, nF, SR, P, seed=41, unvoiced_fraction=0.05)
    dense, _ = syn.make_ctrl(B, nF, SM, seed=42)
    rows = (3, 40)
    noise = torch.zeros(B, nF * P)
    for r in rows:
        noise[r] = syn.normal_noise((1, nF * P), 200 + r)[0]
    leaf = dense.to(DEV).requires_grad_(True)
    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=FixedControls(syn.split_views(leaf, SM),
                                                                  torch.zeros(B, nF, 256, device=DEV))).to(DEV)
    signal, _, _ = model(None, f0.to(DEV), None, noise=noise.to(DEV), infer=False)
    st = _stft()
    ddsp_mel = st.get_mel(signal).transpose(1, 2)            # reflow/vocoder.py extract(): [B, F, n_mels]
    g = torch.Generator().manual_seed(43)
    target = (ddsp_mel.detach().cpu() + 0.3 * torch.randn(ddsp_mel.shape, generator=g))
    W = 1e-3 * torch.randn(ddsp_mel.shape, generator=g)
    loss = torch.nn.functional.mse_loss(ddsp_mel, target.to(DEV)) + (ddsp_mel * W.to(DEV)).sum()
    loss.backward()
    assert torch.isfinite(leaf.grad).all()
    n_total = ddsp_mel.numel()
    for r in rows:
        lr = dense[r:r + 1].clone().requires_grad_(True)
        sig = tp.superfast_forward(f0[r:r + 1], syn.split_views(lr, SM), SR, P, WIN, noise=noise[r:r + 1])["signal"]
        m = om.get_mel(sig).transpose(1, 2)
        (((m - target[r:r + 1]) ** 2).sum() / n_total + (m * W[r:r + 1]).sum()).backward()
        got, want = leaf.grad[r].cpu().double().numpy(), lr.grad[0].double().numpy()
        errs = {k: util.rms(got[:, i * NB:(i + 1) * NB] - want[:, i * NB:(i + 1) * NB]) /
                util.rms(want[:, i * NB:(i + 1) * NB]) for i, k in enumerate(SM)}
        report.record("mel_backward/chain_row%d" % r, **errs)
        for k, v in errs.items():
            assert v <= 5e-4, (r, k, v)


class _LinearControls(torch.nn.Module):
    """a small trainable unit2ctrl: Linear(units) -> split_to_dict (reference ddsp/unit2control.py:12-23)"""

    def __init__(self, n_in, bias):
        super().__init__()
        self.lin = torch.nn.Linear(n_in, 4 * NB)
        with torch.no_grad():
            self.lin.weight.mul_(0.1)
            self.lin.bias.copy_(bias)

    def forward(self, units, f0, phase, volume, **kw):
        return syn.split_views(self.lin(units), SM), None


def test_adam_lowers_the_mel_loss():
    """20 Adam steps on the mel MSE against a teacher's mel; the same loop with the oracle port + oracle.mel on CPU
    goes from 0.278 to 0.020"""
    B, nF, n_in = 2, 40, 16
    f0 = syn.make_f0(B, nF, SR, P, seed=31).to(DEV)
    units = torch.randn(B, nF, n_in, generator=torch.Generator().manual_seed(32)).to(DEV)
    noise = syn.normal_noise((B, nF * P), 33).to(DEV)
    means = torch.tensor([-2.0] * NB + [0.0] * NB + [-3.0] * NB + [0.0] * NB)
    torch.manual_seed(34)
    u2c = _LinearControls(n_in, means)
    torch.manual_seed(35)
    teacher = _LinearControls(n_in, means + 0.5)
    st = _stft()
    with torch.no_grad():
        tm = CombSubSuperFast(SR, P, WIN, unit2ctrl=teacher).to(DEV)
        target = st.get_mel(tm(units, f0, None, noise=noise)[0])
    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=u2c).to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        signal, _, _ = model(units, f0, None, noise=noise, infer=False)
        loss = torch.nn.functional.mse_loss(st.get_mel(signal), target)
        loss.backward()
        assert u2c.lin.weight.grad is not None and u2c.lin.weight.grad.abs().sum() > 0
        opt.step()
        losses.append(loss.item())
    report.record("mel_backward/adam", first=losses[0], last=losses[-1])
    assert np.isfinite(losses).all() and losses[-1] < 0.25 * losses[0], losses
