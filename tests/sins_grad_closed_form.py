"""Float64 restatement of the Sins backward (training phase) with respect to its three raw controls.

TEST INFRASTRUCTURE ONLY.  The independent ground truth of the gradient, as oracle/closed_form.py is for the forward:
the reference's own autograd gradient (tests/golden/sins_grad_*.npz), the oracle port under autograd and the CUDA
kernels must all sit within tolerance of it.  It uses oracle.closed_form for the forward quantities (activated
amplitudes, impulse responses) and numpy's rfft; the three adjoints are written out here:

* FIR (ddsp/core.py:120-182), direct form y[n] = sum_tau ((1 - phi_m) h_f[tau] + phi_m h_{f+1}[tau]) x[m],
  m = n + L/2 - tau, h_nF := h_{nF-1}:
    dh_f[tau] = sum_m w_f(m) x[m] g[m - L/2 + tau],  w_f = 1 - phi on hop f, phi on hop f-1 (and 1 on the last hop),
    dx[m]     = sum_tau ((1 - phi_m) h_f[tau] + phi_m h_{f+1}[tau]) g[m - L/2 + tau];
* impulse responses (ddsp/core.py:254-270): dr = dh un-rolled (noise: times the Hann window first);
  dH_j = c_j rfft(dr)_j with c_j = 2/N (1/N and a real part only at DC and Nyquist: the adjoint of torch's c2r irfft);
  all-pass: dphi_j = Im(dH_j conj(H_j)), reverse cumsum over bins, * pi (1 - tanh^2 c);  noise: Re(dH) exp(c)/128;
* oscillator bank (ddsp/vocoder.py:580-594): dA[k, h] = sum_t dx(t) sin(h phase(t)) w_k(t), w_k the linear-upsample
  hat (the held row nF folded into row nF-1), dc = dA * A.
"""
import numpy as np

from oracle import closed_form as cf


def _sin_args(x32, H, reference_rounding):
    """[B, T, H] arguments of sin: the reference forms fp32(2 pi) * x in fp32 and multiplies by h in fp32
    (ddsp/vocoder.py:574,590); reference_rounding=False: 2 pi h x exactly."""
    h = np.arange(1, H + 1)
    if reference_rounding:
        phase = (np.float32(2 * np.pi) * np.asarray(x32, np.float32)).astype(np.float32)
        return (phase[..., None] * h.astype(np.float32)).astype(np.float32).astype(np.float64)
    return 2 * np.pi * np.asarray(x32, np.float64)[..., None] * h


def kernel_phase(f0_frames, sr, P):
    """[B, T] fp32 wrapped phase in cycles that the training-phase kernels evaluate (DESIGN §4.1): the closed form of
    the cumsum in float64, rounded to fp32 before wrapping.  It differs from the reference's fp32 cumsum by about an
    ulp of x, which sin(2 pi h x) amplifies by 2 pi h: each side is compared with float64 at its own phase."""
    f = np.asarray(f0_frames, np.float64)[..., 0]
    B, nF = f.shape
    fn = np.concatenate([f[:, 1:], f[:, -1:]], axis=1)
    d = fn - f
    S = np.concatenate([np.zeros((B, 1)), np.cumsum((P * f + d * 0.5 * (P - 1)) / sr, axis=1)[:, :-1]], axis=1)
    j = np.arange(P, dtype=np.float64)[None, None, :]
    x = S[:, :, None] + ((j + 1) * f[:, :, None] + d[:, :, None] * (j * (j + 1)) * (0.5 / P)) * (1.0 / sr)
    x = x.astype(np.float32).astype(np.float64)
    return (x - np.rint(x)).astype(np.float32).reshape(B, -1)


def sinusoids(f0_frames, c_amp, x32, sr, P, reference_rounding=True):
    """the oscillator bank in float64 at the phase x32 [B, T]"""
    A = cf.harmonic_amplitudes(np.asarray(c_amp, np.float64), f0_frames, sr)
    B, nF, H = A.shape
    S = np.sin(_sin_args(np.asarray(x32).reshape(B, nF * P), H, reference_rounding))
    return (S * cf.upsample(A, P)).sum(-1)


def _fir_adjoint(x, ir, g, P, want_dx):
    """dh [B, nF, L] (and dx [B, T]) of y = ltv_fir(x, ir) for the cotangent g, all float64."""
    B, nF, L = ir.shape
    T = nF * P
    half = L // 2
    pad = P + half
    gp = np.zeros((B, T + 2 * pad + L))
    gp[:, pad:pad + T] = g                           # gp[pad + n] = g[n]
    phi = np.arange(P) / P
    xh = x.reshape(B, nF, P)
    dh = np.zeros((B, nF, L))
    dx = np.zeros((B, T)) if want_dx else None
    for b in range(B):
        for f in range(nF):
            v = np.zeros(2 * P)
            if f >= 1:
                v[:P] = phi * xh[b, f - 1]
            v[P:] = (1.0 if f == nF - 1 else 1 - phi) * xh[b, f]
            start = pad + (f - 1) * P - half
            dh[b, f] = np.correlate(gp[b, start:start + 2 * P + L - 1], v, "valid")
            if want_dx:
                s = pad + f * P - half
                win = gp[b, s:s + P + L - 1]
                a = np.correlate(win, ir[b, f], "valid")
                c = np.correlate(win, ir[b, min(f + 1, nF - 1)], "valid")
                dx[b, f * P:(f + 1) * P] = (1 - phi) * a + phi * c
    return dh, dx


def _irfft_adjoint(dr):
    """adjoint of torch's c2r irfft (n = N even) applied to dr [..., N] -> complex [..., N/2 + 1]"""
    N = dr.shape[-1]
    R = np.fft.rfft(dr, axis=-1)
    w = np.full(N // 2 + 1, 2.0 / N)
    w[0] = w[-1] = 1.0 / N
    dH = R * w
    dH[..., 0] = dH[..., 0].real
    dH[..., -1] = dH[..., -1].real
    return dH


def sins_grad(f0_frames, ctrls, x32, sr, P, noise, cot, cot_h=None, cot_n=None, reference_rounding=True,
              sinusoids_in=None):
    """Gradient of sum(signal cot + harmonic cot_h + noise cot_n) through Sins (infer=False) with respect to the three
    raw controls, in float64.  ``x32`` [B, T]: the wrapped phase in cycles (the reference's fp32 cumsum; data, not
    differentiated).  ``sinusoids_in`` [B, T]: the all-pass filter's input if not the bank's float64 output (the
    adjoint of a forward that produced these).  Returns {control name: [B, nF, C]}."""
    c = {k: np.asarray(v, np.float64) for k, v in ctrls.items()}
    B, nF, H = c["amplitudes"].shape
    T = nF * P
    cot = np.asarray(cot, np.float64)
    g_h = cot + (0 if cot_h is None else np.asarray(cot_h, np.float64))
    g_n = cot + (0 if cot_n is None else np.asarray(cot_n, np.float64))
    A = cf.harmonic_amplitudes(c["amplitudes"], f0_frames, sr)                    # [B, nF, H]
    S = np.sin(_sin_args(np.asarray(x32).reshape(B, T), H, reference_rounding))   # [B, T, H]
    sinusoids = (S * cf.upsample(A, P)).sum(-1) if sinusoids_in is None else np.asarray(sinusoids_in, np.float64)
    ir_ap = cf.impulse_response(cf.allpass_spectrum(c["group_delay"]), "none")
    ir_n = cf.impulse_response(np.exp(c["noise_magnitude"]) / 128.0, "hann")

    # all-pass filter and its impulse response
    dh, dx = _fir_adjoint(sinusoids, ir_ap, g_h, P, True)
    La = dh.shape[-1]
    dH = _irfft_adjoint(np.roll(dh, -(La // 2), axis=-1))
    phi = np.cumsum(np.pi * np.tanh(c["group_delay"]), axis=-1)
    dphi = (dH * np.exp(-1j * phi)).imag
    d_gd = np.cumsum(dphi[..., ::-1], axis=-1)[..., ::-1] * np.pi * (1 - np.tanh(c["group_delay"]) ** 2)

    # noise filter and its impulse response
    dhn, _ = _fir_adjoint(np.asarray(noise, np.float64), ir_n, g_n, P, False)
    Ln = dhn.shape[-1]
    hann = 0.5 * (1 - np.cos(2 * np.pi * np.arange(Ln) / Ln))
    dHn = _irfft_adjoint(np.roll(dhn * hann, -(Ln // 2), axis=-1))
    d_nm = dHn.real * np.exp(c["noise_magnitude"]) / 128.0

    # oscillator bank
    Y = (dx[:, :, None] * S).reshape(B, nF, P, H)
    lam = (np.arange(P) / P)[None, None, :, None]
    dA = (Y * (1 - lam)).sum(2)
    carry = (Y * lam).sum(2)                  # hop k's weight on row k + 1 (row nF is row nF - 1 held)
    dA[:, 1:] += carry[:, :-1]
    dA[:, -1] += carry[:, -1]
    return {"amplitudes": dA * A, "group_delay": d_gd, "noise_magnitude": d_nm}
