"""Float64 restatement of the random-scale spectral loss (ddsp/loss.py:9-54) and of its gradient with respect to the
prediction, written from the formulas rather than through autograd (numpy only):

    S = |rfft(w frame)| / c + eps            frames at hop n, c = sqrt(sum w^2), K = n // 2 + 1
    D = S_t - S_p,  A = S_t + S_p
    g_S = (1/n_scale) [ (1/B)(-D / (|D| |A|) - |D| A / |A|^3) - alpha sign(log S_t - log S_p) / (B K F S_p) ]
    G = g_S X / (c |X|)  (0 where |X| = 0),   dx[m] = w[m] Re sum_{k<K} G[k] e^{+2 pi i k m / n}

with torch's conventions: sign(0) = 0, the norm's gradient is 0 where the norm is 0, |.|'s gradient is 0 at 0.
tests/test_oracle_rss_loss.py checks it against float64 autograd of oracle.loss to 1e-12.
"""
import numpy as np


def hann(n):
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n) / n)


def _frames(x, n):
    B, T = x.shape
    F = 1 + (T - n) // n
    return x[:, :F * n].reshape(B, F, n), F


def loss_and_grad(x_pred, x_true, n_ffts, alpha=1.0, eps=1e-7):
    """-> (loss, dL/dx_pred [B, T], per-scale norms [n_scale, B, 2]) in float64"""
    xp = np.asarray(x_pred, np.float64)
    xt = np.asarray(x_true, np.float64)
    B, T = xp.shape
    ns = len(n_ffts)
    loss, grad, norms = 0.0, np.zeros_like(xp), np.zeros((ns, B, 2))
    for s, n in enumerate(int(v) for v in n_ffts):
        w = hann(n)
        c = np.sqrt(np.sum(w * w))
        fp, F = _frames(xp, n)
        ft, _ = _frames(xt, n)
        Xp = np.fft.rfft(fp * w, axis=-1) / c
        Xt = np.fft.rfft(ft * w, axis=-1) / c
        K = n // 2 + 1
        Sp, St = np.abs(Xp) + eps, np.abs(Xt) + eps
        D, A = St - Sp, St + Sp
        nD = np.sqrt(np.sum(D * D, axis=(1, 2)))
        nA = np.sqrt(np.sum(A * A, axis=(1, 2)))
        norms[s, :, 0], norms[s, :, 1] = nD, nA
        lt, lp = np.log(St), np.log(Sp)
        loss += np.mean(nD / nA) + alpha * np.mean(np.abs(lt - lp))
        inv = np.where(nD > 0, 1.0 / np.where(nD > 0, nD * nA, 1.0), 0.0)[:, None, None]
        gS = (-D * inv - (nD / nA ** 3)[:, None, None] * A) / B - alpha * np.sign(lt - lp) / (B * K * F * Sp)
        gS /= ns
        mag = np.abs(Xp)
        G = np.where(mag > 0, gS / np.where(mag > 0, mag, 1.0) / c, 0.0) * Xp
        Gpad = np.zeros((B, F, n), np.complex128)
        Gpad[..., :K] = G
        d = np.real(n * np.fft.ifft(Gpad, axis=-1)) * w
        grad[:, :F * n] += d.reshape(B, F * n)
    return loss / ns, grad, norms
