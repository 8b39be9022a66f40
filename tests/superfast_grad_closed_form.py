"""Float64 restatement of the CombSubSuperFast backward with respect to its four raw controls.

TEST INFRASTRUCTURE ONLY.  The independent ground truth of the gradient, as oracle/closed_form.py is for the forward:
the reference's own autograd gradient (tests/golden/superfast_grad_*.npz), the oracle port under autograd and the CUDA
kernel must all sit within tolerance of it.  It shares no code with the port or the kernel apart from
oracle.closed_form.stft_frames (numpy's rfft).
"""
import numpy as np

from oracle.closed_form import stft_frames


def superfast_comb32(f0_frames, sr, P):
    """The comb source of fast_source_gen with the reference's fp32 operation order (ddsp/vocoder.py:639-651).
    The phase is fp32 and the sinc argument divides it by s ~ 1e-3, so the fp32 rounding of the phase is part of
    the signal the reference filters: a gradient with respect to the filters is only comparable at the fp32 floor
    when it uses this source.  Only sin() is evaluated in float64 (of the fp32 product pi*z, as torch.sinc forms it)."""
    f32 = np.float32
    s = (np.asarray(f0_frames, f32)[..., 0] / f32(sr)).astype(f32)
    ds = np.zeros_like(s)
    ds[:, :-1] = s[:, 1:] - s[:, :-1]
    j = np.arange(P, dtype=f32)[None, None, :]
    rad = s[:, :, None] * (j + f32(1))
    rad = rad + (((f32(0.5) * ds)[:, :, None] * j) * (j + f32(1))) / f32(P)
    s_up = s[:, :, None] + (ds[:, :, None] * j) / f32(P)
    adv = np.fmod(rad[:, :, -1] + f32(0.5), f32(1.0)) - f32(0.5)
    acc = np.fmod(np.cumsum(adv.astype(np.float64), axis=1).astype(f32), f32(1.0))     # fp64 accumulation
    rad = rad + np.concatenate([np.zeros((s.shape[0], 1), f32), acc[:, :-1]], axis=1)[:, :, None]
    rad = rad - np.rint(rad)
    z = rad / (s_up + f32(1e-5))
    pz = (f32(np.pi) * z).astype(f32)
    with np.errstate(invalid="ignore", divide="ignore"):
        comb = np.where(z == 0, 1.0, np.sin(pz.astype(np.float64)) / pz.astype(np.float64))
    return comb.reshape(s.shape[0], -1)


def superfast_grad(f0_frames, ctrls, sr, P, win_length, noise, grad_signal, comb=None):
    """Gradient of sum(superfast(...)["signal"] * grad_signal) with respect to the four raw controls, in float64.

    With g = grad_signal, N = win_length, win the periodic Hann window and env the OLA(win^2) the iSTFT divides by,
    for every STFT frame q = 0..nF (frame nF holds control row nF-1):
      r_q[i] = win[i] g[n] / env(n), n = qP + i - N/2 (zero outside [0, T): the part the iSTFT trims)
      G_q    = (2/N) rfft(r_q)[k] for 0 < k < N/2;  (1/N) Re rfft(r_q)[k] at k = 0, N/2 (irfft ignores Im there)
      A      = X_q exp(m_h + j pi p_h)   (noise: N_q exp(m_n + j pi p_n) / 128)
      dL/dm  = Re(conj(G_q) A),  dL/dp = -pi Im(conj(G_q) A),  frame nF added into row nF-1.
    ``comb``: the source; default superfast_comb32 (the reference's fp32 source).
    Returns {control name: [B, nF, N/2+1]}."""
    if comb is None:
        comb = superfast_comb32(f0_frames, sr, P)
    comb = np.asarray(comb, np.float64)
    B, T = comb.shape
    nF, N, half = T // P, win_length, win_length // 2
    mode = "reflect" if T > half else "constant"
    X = stft_frames(comb, N, P, mode)
    Nz = stft_frames(np.asarray(noise, np.float64), N, P, mode)
    win = 0.5 * (1 - np.cos(2 * np.pi * np.arange(N) / N))
    total = N + P * nF
    env = np.zeros(total)
    for q in range(nF + 1):
        env[q * P:q * P + N] += win * win
    gp = np.zeros((B, total))
    gp[:, half:half + T] = np.asarray(grad_signal, np.float64) / env[half:half + T]
    idx = np.arange(N)[None, :] + P * np.arange(nF + 1)[:, None]
    R = np.fft.rfft(gp[:, idx] * win, axis=-1)
    Gq = (2.0 / N) * R
    Gq[..., 0] = R[..., 0].real / N
    Gq[..., half] = R[..., half].real / N
    hold = lambda z: np.concatenate([z, z[:, -1:, :]], axis=1)
    c = {k: np.asarray(v, np.float64) for k, v in ctrls.items()}
    Ah = X * hold(np.exp(c["harmonic_magnitude"] + 1j * np.pi * c["harmonic_phase"]))
    An = Nz * hold(np.exp(c["noise_magnitude"] + 1j * np.pi * c["noise_phase"]) / 128.0)

    def fold(d):
        out = d[:, :nF].copy()
        out[:, nF - 1] += d[:, nF]
        return out

    pa, pn = np.conj(Gq) * Ah, np.conj(Gq) * An
    return {"harmonic_magnitude": fold(pa.real), "harmonic_phase": fold(-np.pi * pa.imag),
            "noise_magnitude": fold(pn.real), "noise_phase": fold(-np.pi * pn.imag)}
