"""Float64 restatement of the old-CombSub backward (training phase) with respect to its three raw controls.

TEST INFRASTRUCTURE ONLY.  The independent ground truth of the gradient: the reference's own autograd gradient
(tests/golden/combsub_grad_*.npz), the oracle port under autograd and the CUDA kernels must all sit within tolerance
of it.  It uses oracle.closed_form for the forward quantities and the FIR / irfft adjoints of
tests/sins_grad_closed_form.py; the cascade and the dynamic window are written out here:

* a = FIR(comb, h_ap), harmonic = FIR(a, h_h), noise = FIR(u, h_n)  (ddsp/vocoder.py:846-862);
* harmonic filter: dh_h = corr(g_h, a), da = FIR^T(g_h, h_h); dr = dh_h times the per-frame dynamic window
  w = (1 + cos(pi u)) / 2, u = (tau - L/2) / (1.5 sr / (f0 + 1e-3)), u := 0 where u > 1 (ddsp/core.py:240-251),
  un-rolled; dc_h = Re(dH) exp(c_h);
* noise filter: as Sins, dc_n = Re(dH) exp(c_n) / 128;
* all-pass filter on the comb with the cotangent da: dphi_j = Im(dH_j conj H_j), reverse cumsum, * pi (1 - tanh^2 c).

The comb is an input: in the training phase it depends on how the phase was rounded to fp32 (the reference rounds its
fp32 cumsum, the kernels the closed-form fp64 phase), and sinc amplifies a phase ulp by sr / f0.  Feeding each
implementation's own comb separates that source difference from the backward.
"""
import numpy as np

from oracle import closed_form as cf
from tests.sins_grad_closed_form import _fir_adjoint, _irfft_adjoint


def dynamic_window(f0_frames, sr, L):
    """[B, nF, L] the per-frame raised cosine of the harmonic impulse response, in float64"""
    hw = 1.5 * sr / (np.asarray(f0_frames, np.float64).reshape(-1, np.shape(f0_frames)[1], 1) + 1e-3)
    u = (np.arange(L, dtype=np.float64) - L // 2) / hw
    u = np.where(u > 1, 0.0, u)
    return 0.5 * (1 + np.cos(np.pi * u))


def combsub_grad(f0_frames, ctrls, comb, sr, P, noise, cot, cot_h=None, cot_n=None, allpassed_in=None):
    """Gradient of sum(signal cot + harmonic cot_h + noise cot_n) through CombSub (infer=False) with respect to the
    three raw controls, in float64.  ``comb`` [B, T]: the comb source (data).  ``allpassed_in`` [B, T]: the harmonic
    filter's input if not the float64 all-pass of ``comb``.  Returns {control name: [B, nF, C]}."""
    c = {k: np.asarray(v, np.float64) for k, v in ctrls.items()}
    comb = np.asarray(comb, np.float64)
    cot = np.asarray(cot, np.float64)
    g_h = cot + (0 if cot_h is None else np.asarray(cot_h, np.float64))
    g_n = cot + (0 if cot_n is None else np.asarray(cot_n, np.float64))
    ir_ap = cf.impulse_response(cf.allpass_spectrum(c["group_delay"]), "none")
    Lh = 2 * (c["harmonic_magnitude"].shape[-1] - 1)
    win = dynamic_window(f0_frames, sr, Lh)
    ir_h = cf.impulse_response(np.exp(c["harmonic_magnitude"]), "none") * win
    ir_n = cf.impulse_response(np.exp(c["noise_magnitude"]) / 128.0, "hann")
    allpassed = cf.ltv_fir(comb, ir_ap, P) if allpassed_in is None else np.asarray(allpassed_in, np.float64)

    # harmonic filter: its impulse response and the cascade's input gradient
    dh, da = _fir_adjoint(allpassed, ir_h, g_h, P, True)
    dHh = _irfft_adjoint(np.roll(dh * win, -(Lh // 2), axis=-1))
    d_hm = dHh.real * np.exp(c["harmonic_magnitude"])

    # all-pass filter on the comb, cotangent da
    dha, _ = _fir_adjoint(comb, ir_ap, da, P, False)
    La = dha.shape[-1]
    dH = _irfft_adjoint(np.roll(dha, -(La // 2), axis=-1))
    phi = np.cumsum(np.pi * np.tanh(c["group_delay"]), axis=-1)
    dphi = (dH * np.exp(-1j * phi)).imag
    d_gd = np.cumsum(dphi[..., ::-1], axis=-1)[..., ::-1] * np.pi * (1 - np.tanh(c["group_delay"]) ** 2)

    # noise filter
    dhn, _ = _fir_adjoint(np.asarray(noise, np.float64), ir_n, g_n, P, False)
    Ln = dhn.shape[-1]
    hann = 0.5 * (1 - np.cos(2 * np.pi * np.arange(Ln) / Ln))
    dHn = _irfft_adjoint(np.roll(dhn * hann, -(Ln // 2), axis=-1))
    d_nm = dHn.real * np.exp(c["noise_magnitude"]) / 128.0
    return {"group_delay": d_gd, "harmonic_magnitude": d_hm, "noise_magnitude": d_nm}


def kernel_comb(f0_frames, sr, P):
    """[B, T] the comb of the training-phase kernels in float64: sinc at their fp32 phase (DESIGN §4.1)"""
    from tests.sins_grad_closed_form import kernel_phase
    x32 = kernel_phase(f0_frames, sr, P).astype(np.float64)
    f0_up = cf.upsample(f0_frames, P)[..., 0]
    return np.sinc(sr * x32 / (f0_up + 1e-3))
