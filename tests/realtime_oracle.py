"""Float64 statement of gui.py's real-time block around the networks (reference gui.py:15-31, :434-454,
ddsp/vocoder.py:108-118 and :138-144, enhancer.py:65-70), written without np.interp, np.fft or np.correlate so that
tests/test_realtime.py can check it against those independent formulations.  fp32 appears only where the reference
stores into an fp32 array or tensor."""
import numpy as np


def interp(x, xp, fp):
    """np.interp(x, xp, fp) for increasing xp: (fp[i+1] - fp[i]) / (xp[i+1] - xp[i]) (x - xp[i]) + fp[i] on the
    interval xp[i] <= x < xp[i+1], fp[0] left of xp[0], fp[-1] at or right of xp[-1]"""
    x, xp, fp = np.asarray(x, np.float64), np.asarray(xp, np.float64), np.asarray(fp, np.float64)
    out = np.empty(x.shape)
    for j, v in enumerate(x.ravel()):
        if v < xp[0]:
            out.flat[j] = fp[0]
        elif v >= xp[-1]:
            out.flat[j] = fp[-1]
        else:
            i = int(np.sum(xp <= v)) - 1
            out.flat[j] = fp[i] if xp[i] == v else (fp[i + 1] - fp[i]) / (xp[i + 1] - xp[i]) * (v - xp[i]) + fp[i]
    return out


def fill_unvoiced(f):
    """zero frames replaced by the linear interpolation of their voiced neighbours (held past the first / last voiced
    frame); unchanged when no frame is voiced.  The result has f's dtype, as an in-place numpy assignment has."""
    f = np.array(f)
    voiced = np.flatnonzero(f != 0)
    if len(voiced) == 0:
        return f
    for i in np.flatnonzero(f == 0):
        if i < voiced[0]:
            f[i] = f[voiced[0]]
        elif i > voiced[-1]:
            f[i] = f[voiced[-1]]
        else:
            q = voiced[np.searchsorted(voiced, i)]
            p = voiced[np.searchsorted(voiced, i) - 1]
            f[i] = (np.float64(f[q]) - np.float64(f[p])) / (q - p) * (i - p) + np.float64(f[p])
    return f


def rmvpe_f0(f0_10ms, hop_size, sample_rate, n_frames, start_frame, f0_min, pitch_adjust=0.0):
    """F0_Extractor('rmvpe').extract(..., uv_interp=True) after RMVPE, then SvcDDSP.infer's .float() and pitch factor:
    f0_10ms float32 [n] (0 = unvoiced) -> float32 [n_frames]"""
    f0 = np.asarray(f0_10ms, np.float32)
    uv = f0 == 0
    filled = fill_unvoiced(f0)                                          # float32, as the reference's array
    src = 0.01 * np.arange(len(f0))
    dst = hop_size / sample_rate * np.arange(n_frames - start_frame)
    g = interp(dst, src, filled)
    g[interp(dst, src, uv.astype(np.float64)) > 0.5] = 0
    g = np.concatenate([np.zeros(start_frame), g])
    g = fill_unvoiced(g)
    g[g < f0_min] = f0_min
    return g.astype(np.float32) * np.float32(2 ** (float(pitch_adjust) / 12))


def adaptive_rate(enhancer_sample_rate, adaptive_key):
    """Enhancer.enhance's adaptive sample rate and real_factor for a numeric key"""
    factor = 2 ** (-float(adaptive_key) / 12)
    rate = 100 * int(np.round(enhancer_sample_rate / factor / 100))
    return rate, enhancer_sample_rate / rate


def enhancer_f0(f0, hop_size, sample_rate, real_factor, enhancer_hop, enhancer_rate, n_frames, start_frame=0):
    """Enhancer.enhance's f0 resampling: f0 float32 [n] -> float32 [n_frames]"""
    f = np.asarray(f0, np.float32)[start_frame:] * np.float32(real_factor)
    src = (hop_size / sample_rate) * np.arange(len(f)) / real_factor
    dst = (enhancer_hop / enhancer_rate) * np.arange(n_frames)
    return interp(dst, src, f).astype(np.float32)


def sola_scores(x, buf, search):
    """gui.py's cor_nom / cor_den for shifts 0..search, float64"""
    x, buf = np.asarray(x, np.float64), np.asarray(buf, np.float64)
    n = len(buf)
    return np.array([np.dot(x[s:s + n], buf) / np.sqrt(np.dot(x[s:s + n], x[s:s + n]) + 1e-8)
                     for s in range(search + 1)])


def fade_windows(crossfade):
    """start_vc's windows in float64: sin(pi t / 2)^2 on torch.arange(0, 1, 1 / crossfade), and 1 minus it"""
    t = np.arange(crossfade) / crossfade
    fade_in = np.sin(np.pi * t / 2) ** 2
    return fade_in, 1 - fade_in


def phase_vocoder(a, b, fade_out, fade_in):
    """gui.py's phase_vocoder in float64 with a direct DFT and synthesis sum, the phase k t reduced mod n in integers"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    fade_out, fade_in = np.asarray(fade_out, np.float64), np.asarray(fade_in, np.float64)
    n = len(a)
    w = np.sqrt(fade_out * fade_in)
    k = np.arange(n // 2 + 1)
    t = np.arange(n)
    ang = 2 * np.pi * ((k[:, None] * t[None]) % n) / n                 # [bins, n]
    fa = (a * w) @ np.exp(-1j * ang).T
    fb = (b * w) @ np.exp(-1j * ang).T
    amp = np.abs(fa) + np.abs(fb)
    amp[1:(n - 1) // 2 + 1] *= 2
    pa = np.angle(fa)
    d = np.angle(fb) - pa
    d = d - 2 * np.pi * np.floor(d / 2 / np.pi + 0.5)
    phase = ang.T + d[None] * (t[:, None] / n) + pa[None]               # [n, bins]
    return a * fade_out ** 2 + b * fade_in ** 2 + np.sum(amp * np.cos(phase), -1) * w / n


def crossfade(x, shift, buf, fade_in, fade_out, block, use_phase_vocoder):
    """gui.py:441-456 at a given shift -> (out [block], next sola buffer [crossfade]), float64"""
    cf = len(buf)
    y = np.array(x[shift:shift + block + cf], np.float64)
    if use_phase_vocoder:
        y[:cf] = phase_vocoder(buf, y[:cf], fade_out, fade_in)
    else:
        y[:cf] = y[:cf] * fade_in + np.asarray(buf, np.float64) * fade_out
    return y[:block], y[block:]
