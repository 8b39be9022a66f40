"""The gradient oracles of Sins (training phase) against the reference's own autograd gradient (CPU).

tests/golden/sins_grad_*.npz hold dense.grad of the live reference (make_golden_sins_grad.py).
* oracle.torch_port.sins_forward(infer=False) under autograd runs the reference's ATen operators, so its gradient must
  be bit-identical; that licenses the port as the gradient oracle for shapes too large for goldens;
* tests/sins_grad_closed_form.sins_grad restates the backward in float64: it must match float64 autograd of the same
  math to ~1e-12, and the goldens at the fp32 floor."""
import math

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import synthetic as syn
from oracle import torch_port as tp
from tests import sins_grad_closed_form as cfg
from tests import util
from tests.golden import make_golden_sins_grad as GG

NAMES = list(GG.CASES)
KEYS = ("amplitudes", "group_delay", "noise_magnitude")


def load(name):
    inp = GG.build_inputs(name)
    z = np.load(GG.path(name), allow_pickle=False)
    gold = {k: z[k] for k in z.files}
    for k, v in GG.input_checksums(inp).items():
        assert abs(float(gold[k]) - v) <= 1e-9 * max(1.0, abs(v)), "input %s of %s differs from the golden's" % (k, name)
    return inp, gold


def split_grad(name, dense_grad):
    return {k: np.asarray(v, np.float64) for k, v in
            syn.split_views(torch.as_tensor(np.asarray(dense_grad)), GG.split_map(name)).items()}


def rel_rms(got, ref):
    return util.rms(np.asarray(got, np.float64) - ref) / util.rms(ref)


def x32_of(inp):
    """the reference's training-phase wrapped phase (fp32 cumsum, ddsp/vocoder.py:568-572), [B, T]"""
    x, _ = tp.wrapped_phase(inp["f0"], GG.SR, GG.P, infer=False)
    return x[..., 0].numpy()


def closed_form(inp, reference_rounding=True, x32=None):
    """float64 gradient at the reference's phase (default) or at ``x32``"""
    x32 = x32_of(inp) if x32 is None else x32
    return cfg.sins_grad(inp["f0"].numpy(), {k: v.numpy() for k, v in inp["ctrls"].items()}, x32, GG.SR, GG.P,
                         inp["noise"].numpy(), inp["cot"].numpy(),
                         None if inp["cot_h"] is None else inp["cot_h"].numpy(),
                         None if inp["cot_n"] is None else inp["cot_n"].numpy(), reference_rounding)


def error_model(inp, gold_grad, name):
    """-> (truth at the kernels' phase {control: float64 [B, nF, C]}, {control: the fp32 reference's own relative RMS
    error against float64 at ITS phase}).  A kernel result is checked against the first, within a multiple of the
    second (tests/test_emu_sins_backward.py, tests/test_gpu_sins_backward.py)."""
    exact = closed_form(inp, reference_rounding=False)
    gold = split_grad(name, gold_grad)
    ref_err = {k: rel_rms(gold[k], exact[k]) for k in KEYS}
    truth = closed_form(inp, reference_rounding=False, x32=cfg.kernel_phase(inp["f0"].numpy(), GG.SR, GG.P))
    return truth, ref_err


@pytest.mark.parametrize("name", NAMES)
def test_port_autograd_is_bit_identical_to_reference(name):
    inp, gold = load(name)
    dense = inp["dense"].clone().requires_grad_(True)
    out = tp.sins_forward(inp["f0"], syn.split_views(dense, GG.split_map(name)), GG.SR, GG.P, noise=inp["noise"],
                          infer=False)
    assert torch.equal(out["signal"].detach(), torch.from_numpy(gold["signal"]))
    GG.objective(out["signal"], out["harmonic"], out["noise"], inp).backward()
    assert torch.equal(dense.grad, torch.from_numpy(gold["grad"]))


def _f64_forward(dense, name, x32, f0, noise):
    """The same math in float64 under torch autograd (no fp32 rounding anywhere; sin of 2 pi h x exactly)."""
    P, sr = GG.P, GG.SR
    c = syn.split_views(dense, GG.split_map(name))
    H = c["amplitudes"].shape[-1]
    keep = ((f0 * torch.arange(1, H + 1, dtype=torch.float32)) < sr / 2).double() + float(np.float32(1e-7))
    amp = torch.exp(c["amplitudes"]) / 128 * keep
    S = torch.sin(2 * math.pi * torch.from_numpy(np.asarray(x32, np.float64))[..., None] *
                  torch.arange(1, H + 1, dtype=torch.float64))
    sinus = (S * tp.frames_to_samples(amp, P)).sum(-1)

    def ir(spec, hann):
        r = torch.fft.irfft(spec)
        L = r.shape[-1]
        if hann:
            w = 0.5 * (1 - torch.cos(2 * math.pi * torch.arange(L, dtype=torch.float64) / L))
            return r.roll(L // 2, -1) * w
        return r.roll(L // 2, -1)

    harmonic = tp.ltv_fir(sinus, ir(torch.exp(1j * torch.cumsum(math.pi * torch.tanh(c["group_delay"]), -1)), False))
    nm = torch.exp(c["noise_magnitude"]) / 128
    noise_out = tp.ltv_fir(noise, ir(torch.complex(nm, torch.zeros_like(nm)), True))
    return harmonic + noise_out, harmonic, noise_out


@pytest.mark.parametrize("name", NAMES)
def test_closed_form_matches_float64_autograd(name):
    inp, _ = load(name)
    x32 = x32_of(inp)
    dense = inp["dense"].double().requires_grad_(True)
    sig, harm, nz = _f64_forward(dense, name, x32, inp["f0"], inp["noise"].double())
    d = {k: (None if inp[k] is None else inp[k].double()) for k in ("cot", "cot_h", "cot_n")}
    GG.objective(sig, harm, nz, d).backward()
    want = split_grad(name, dense.grad.numpy())
    got = closed_form(inp, reference_rounding=False)
    for k in KEYS:
        e = rel_rms(got[k], want[k])
        assert e <= 1e-11, (name, k, e)


@pytest.mark.parametrize("name", NAMES)
def test_closed_form_gradient_matches_reference(name):
    """fp32 floor: the reference's fp32 FFTs and sums against float64 (relative RMS per control)"""
    inp, gold = load(name)
    got = closed_form(inp)
    ref = split_grad(name, gold["grad"])
    for k in KEYS:
        assert got[k].shape == ref[k].shape
        e = rel_rms(got[k], ref[k])
        assert e <= 2e-5, (name, k, e)
