"""Float64 restatement of the CombSubFast backward with respect to its three raw controls.

TEST INFRASTRUCTURE ONLY.  The independent ground truth of the gradient, as oracle/closed_form.py is for the forward:
the reference's own autograd gradient (tests/golden/csfast_grad_*.npz), the oracle port under autograd and the CUDA
kernel must all sit within tolerance of it.  It uses numpy's rfft and shares no code with the port or the kernel.

The comb source is an input: in the training phase the comb depends on how the phase was rounded to fp32 (the
reference rounds torch's fp64-accumulated cumsum, the kernels round the closed-form fp64 phase), and sinc amplifies a
phase ulp by sr / f0.  Feeding each implementation's own comb separates that source difference from the backward.
"""
import numpy as np


def combsubfast_grad(comb, ctrls, P, noise, grad_signal):
    """Gradient of sum(combsubfast(comb, ...)["signal"] * grad_signal) with respect to the three raw controls.

    With g = grad_signal, N = 2P, w = sqrt(Hann_N) (periodic), for every frame q = 0..nF (frame q covers samples
    [(q-1)P, (q+1)P) and uses control row min(q, nF-1)):
      rho_q[i] = w[i] g[(q-1)P + i]  (zero outside [0, T))
      G_q      = (2/N) rfft(rho_q)[k] for 0 < k < P;  (1/N) Re rfft(rho_q)[k] at k = 0, P (irfft ignores Im there)
      A_q      = rfft(w comb_q) exp(m_h + j pi p_h),  B_q = rfft(w noise_q) exp(m_n) / 128
      dL/dm_h  = Re(conj(G) A),  dL/dp_h = -pi Im(conj(G) A),  dL/dm_n = Re(conj(G) B);  frame nF added into row nF-1.
    comb, noise, grad_signal: [B, T]; ctrls: {name: [B, nF, P+1]}.  Returns {control name: [B, nF, P+1]} (float64)."""
    comb = np.asarray(comb, np.float64)
    B, T = comb.shape
    nF, N = T // P, 2 * P
    w = np.sqrt(0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N))
    idx = np.arange(N)[None, :] + P * np.arange(nF + 1)[:, None]          # padded position of frame q, sample i

    def frames(z):
        return np.pad(np.asarray(z, np.float64), ((0, 0), (P, P)))[:, idx] * w

    C = np.fft.rfft(frames(comb), axis=-1)
    Z = np.fft.rfft(frames(noise), axis=-1)
    R = np.fft.rfft(frames(grad_signal), axis=-1)
    G = (2.0 / N) * R
    G[..., 0] = R[..., 0].real / N
    G[..., P] = R[..., P].real / N
    hold = lambda z: np.concatenate([z, z[:, -1:, :]], axis=1)
    c = {k: np.asarray(v, np.float64) for k, v in ctrls.items()}
    A = C * hold(np.exp(c["harmonic_magnitude"] + 1j * np.pi * c["harmonic_phase"]))
    Bn = Z * hold(np.exp(c["noise_magnitude"]) / 128.0)

    def fold(d):
        out = d[:, :nF].copy()
        out[:, nF - 1] += d[:, nF]
        return out

    pa, pn = np.conj(G) * A, np.conj(G) * Bn
    return {"harmonic_magnitude": fold(pa.real), "harmonic_phase": fold(-np.pi * pa.imag),
            "noise_magnitude": fold(pn.real)}
