"""The spectral losses of ddsp/loss.py:9-54 (single-scale and random-scale) restated on torch.stft, so they run where
torchaudio is absent.  torchaudio.transforms.Spectrogram(n_fft, hop_length, power=1, normalized=True, center=False)
is, in its own operation order (torchaudio.functional.spectrogram):

    spec = torch.stft(x, n_fft, hop, n_fft, hann_window(n_fft), center=False, normalized=False, onesided=True)
    spec /= window.pow(2.).sum().sqrt();  |spec|

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Bit-identical to the reference on CPU
(tests/test_oracle_rss_loss.py checks the goldens made by the reference's own module).
"""
import torch
import torch.nn.functional as F


def spectrogram(x, n_fft, hop_length, window=None):
    """torchaudio Spectrogram(power=1, normalized=True, center=False) of x [..., T] -> [..., n_fft // 2 + 1, frames]"""
    if window is None:
        window = torch.hann_window(n_fft, device=x.device, dtype=x.dtype)
    shape = x.size()
    x = x.reshape(-1, shape[-1])
    spec = torch.stft(input=x, n_fft=n_fft, hop_length=hop_length, win_length=n_fft, window=window, center=False,
                      pad_mode="reflect", normalized=False, onesided=True, return_complex=True)
    spec = spec.reshape(shape[:-1] + spec.shape[-2:])
    spec /= window.pow(2.0).sum().sqrt()
    return spec.abs()


def scale_loss(x_pred, x_true, n_fft, alpha=1.0, overlap=0, eps=1e-7):
    """the loss at one scale: spectral convergence (per row ||S_t - S_p|| / ||S_t + S_p||, averaged over rows) plus
    alpha times the mean absolute log-magnitude difference, with S = spectrogram + eps (target spectrum taken first,
    as the reference does; the order fixes the rounding)"""
    hop = int(n_fft * (1 - overlap))
    mag_t = spectrogram(x_true, n_fft, hop) + eps
    mag_p = spectrogram(x_pred, n_fft, hop) + eps
    dims = (1, 2)
    convergence = torch.mean(torch.linalg.norm(mag_t - mag_p, dim=dims) / torch.linalg.norm(mag_t + mag_p, dim=dims))
    return convergence + alpha * F.l1_loss(mag_t.log(), mag_p.log())


def rss_loss(x_pred, x_true, n_ffts, alpha=1.0, overlap=0, eps=1e-7):
    """the random-scale loss with its scales ``n_ffts`` already drawn: the scale losses accumulated in draw order onto
    a Python 0.0, divided by the number of scales"""
    total = 0.
    for n in n_ffts:
        total = total + scale_loss(x_pred, x_true, int(n), alpha, overlap, eps)
    return total / len(n_ffts)


def draw_scales(fft_min, fft_max, n_scale):
    """the reference's draw, on torch's default CPU generator"""
    return torch.randint(fft_min, fft_max, (n_scale,))
