"""Log-mel front end of the NSF-HiFiGAN vocoder on the GPU: drop-in for nsf_hifigan.nvSTFT.STFT (reference
nsf_hifigan/nvSTFT.py:59-122), the consumer of the synthesizer's waveform in enhancer.py:113, diffusion/vocoder.py:147
and reflow/vocoder.py:125 (SURVEY 8f rank 4).

``STFT.get_mel(y)`` runs ONE kernel (csrc/mel.cu: padding + Hann frames + 2048-point FFT + magnitude + sparse mel
projection + log) for the shape every shipped configuration uses -- keyshift 0, speed 1, n_fft = win_size = 2048.
Other shapes raise NotImplementedError (there is no PyTorch fallback in this package).  When ``y`` requires grad (and
grad mode is on), the result is differentiable with respect to ``y``: the backward runs ``mel_bwd_kernel`` (same file),
which recomputes the spectra from ``y`` instead of storing them.

The mel filterbank is librosa's (``librosa.filters.mel``, Slaney scale and normalisation: a third-party dependency of
the reference, unpinned in requirements.txt and absent here); ``mel_filterbank`` restates its published algorithm.
"""
import numpy as np
import torch

from . import _lib
from .ops import _count, _need_cuda_f32, _stream


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, min_log_hz) / min_log_hz) / logstep, mels)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def _hz_to_mel_htk(f):
    return 2595.0 * np.log10(1.0 + np.asarray(f, dtype=np.float64) / 700.0)


def _mel_to_hz_htk(m):
    return 700.0 * (10.0 ** (np.asarray(m, dtype=np.float64) / 2595.0) - 1.0)


def mel_filterbank(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, htk=False):
    """librosa.filters.mel(sr=, n_fft=, n_mels=, fmin=, fmax=, htk=) with norm='slaney': triangular filters with
    corners equally spaced on the Slaney (htk=False, librosa's default) or HTK (2595 log10(1 + f / 700)) mel scale, each
    normalised to unit area -> float32 [n_mels, 1 + n_fft // 2]."""
    to_mel, to_hz = (_hz_to_mel_htk, _mel_to_hz_htk) if htk else (_hz_to_mel, _mel_to_hz)
    fmax = float(sr) / 2 if fmax is None else float(fmax)
    fftfreqs = np.linspace(0.0, float(sr) / 2, 1 + n_fft // 2)
    mel_f = to_hz(np.linspace(to_mel(fmin), to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    lower = -ramps[:-2] / fdiff[:-1, None]
    upper = ramps[2:] / fdiff[1:, None]
    weights = np.maximum(0.0, np.minimum(lower, upper))
    weights *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return weights.astype(np.float32)


def _support(basis):
    """[n_mels, 2] int32: first and one-past-last non-zero bin of each filter (empty filters -> 0, 0)."""
    nz = basis != 0
    lo = np.where(nz.any(1), nz.argmax(1), 0)
    hi = np.where(nz.any(1), basis.shape[1] - nz[:, ::-1].argmax(1), 0)
    return np.stack([lo, hi], 1).astype(np.int32)


def _bin_filters(basis):
    """[n_bins, 2] int32: first and one-past-last filter that is non-zero at each bin (bins no filter covers -> 0, 0);
    the rows of the transposed projection the backward kernel sums over."""
    nz = basis.T != 0
    lo = np.where(nz.any(1), nz.argmax(1), 0)
    hi = np.where(nz.any(1), basis.shape[0] - nz[:, ::-1].argmax(1), 0)
    return np.stack([lo, hi], 1).astype(np.int32)


class STFT:
    def __init__(self, sr=22050, n_mels=80, n_fft=1024, win_size=1024, hop_length=256, fmin=20, fmax=11025, clip_val=1e-5):
        self.target_sr = sr
        self.n_mels = n_mels
        self.n_fft = n_fft
        self.win_size = win_size
        self.hop_length = hop_length
        self.fmin = fmin
        self.fmax = fmax
        self.clip_val = clip_val
        self.mel_basis = {}
        self.hann_window = {}

    def _tables(self, device):
        key = str(self.fmax) + "_" + str(device)
        if key not in self.mel_basis:
            mel = mel_filterbank(self.target_sr, self.n_fft, self.n_mels, self.fmin, self.fmax)
            self.mel_basis[key] = (torch.from_numpy(mel).to(device), torch.from_numpy(_support(mel)).to(device),
                                   torch.from_numpy(_bin_filters(mel)).to(device))
            self.hann_window[key] = torch.hann_window(self.win_size).to(device)
        return self.mel_basis[key] + (self.hann_window[key],)

    def _checked(self, y, keyshift, speed, center):
        """the checked (y, B, T, n_frames) of a get_mel call"""
        if keyshift != 0 or speed != 1 or center:
            raise NotImplementedError("the mel kernel covers keyshift=0, speed=1, center=False (the inference call of "
                                      "enhancer.py:113); got keyshift=%r speed=%r center=%r" % (keyshift, speed, center))
        if self.n_fft != 2048 or self.win_size != 2048 or self.n_mels > 128:
            raise NotImplementedError("the mel kernel is built for n_fft = win_size = 2048 and n_mels <= 128 "
                                      "(the 44.1 kHz NSF-HiFiGAN configuration); got %d / %d / %d" % (self.n_fft, self.win_size, self.n_mels))
        _need_cuda_f32("y", y)
        if y.dim() != 2:
            raise ValueError("y must be [B, n_samples]")
        B, T = y.shape
        n_frames = _lib.lib().b2d_mel_frames(T, self.n_fft, self.win_size, int(self.hop_length))
        if n_frames <= 0:
            raise ValueError("signal of %d samples is too short for one frame" % T)
        return y.contiguous(), B, T, n_frames

    def get_mel(self, y, keyshift=0, speed=1, center=False):
        """y [B, T] CUDA fp32 -> log-mel [B, n_mels, n_frames] (nvSTFT.py:73-117).
        Differentiable with respect to y when y requires grad and grad mode is on (CUDA backward, get_mel_backward)."""
        if torch.is_grad_enabled() and isinstance(y, torch.Tensor) and y.requires_grad:
            self._checked(y, keyshift, speed, center)
            return _GetMel.apply(self, y)
        return self._forward(y, keyshift, speed, center)

    def _forward(self, y, keyshift=0, speed=1, center=False):
        y, B, T, n_frames = self._checked(y, keyshift, speed, center)
        L = _lib.lib()
        basis, lohi, _, window = self._tables(y.device)
        out = torch.empty(B, self.n_mels, n_frames, dtype=torch.float32, device=y.device)
        _lib.check(L.b2d_mel_spectrogram(y.data_ptr(), window.data_ptr(), basis.data_ptr(), lohi.data_ptr(), B, T, self.n_fft,
                                         self.win_size, int(self.hop_length), self.n_mels, float(self.clip_val), out.data_ptr(),
                                         _stream()), "b2d_mel_spectrogram")
        _count(1)
        return out

    def get_mel_backward(self, y, grad_mel):
        """Gradient of get_mel(y) with respect to y for dL/dmel ``grad_mel`` [B, n_mels, n_frames] -> [B, n_samples].
        grad_mel may be any strided view (e.g. the transpose of a [B, n_frames, n_mels] tensor): it is read through its
        strides, not copied.  The spectra are recomputed from y, so y must be the forward's input."""
        y, B, T, n_frames = self._checked(y.detach(), 0, 1, False)
        _need_cuda_f32("grad_mel", grad_mel)
        if tuple(grad_mel.shape) != (B, self.n_mels, n_frames):
            raise ValueError("grad_mel must be [B, n_mels, n_frames] = [%d, %d, %d], got %s"
                             % (B, self.n_mels, n_frames, tuple(grad_mel.shape)))
        if grad_mel.device != y.device:
            raise ValueError("grad_mel lives on %s, y on %s" % (grad_mel.device, y.device))
        basis, lohi, bins, window = self._tables(y.device)
        grad = torch.empty(B, T, dtype=torch.float32, device=y.device)
        sb, sm, sf = grad_mel.stride()
        _lib.check(_lib.lib().b2d_mel_spectrogram_backward(
            y.data_ptr(), window.data_ptr(), basis.data_ptr(), lohi.data_ptr(), bins.data_ptr(), B, T, self.n_fft,
            self.win_size, int(self.hop_length), self.n_mels, float(self.clip_val), grad_mel.data_ptr(), sb, sm, sf,
            grad.data_ptr(), _stream()), "b2d_mel_spectrogram_backward")
        _count(1)
        return grad


class _GetMel(torch.autograd.Function):
    """STFT.get_mel with a CUDA backward.  Saves only y: the backward kernel recomputes the spectra and the mel values
    (bit-identical to the forward's, so it takes the same clamp decisions)."""

    @staticmethod
    def forward(ctx, stft, y):
        ctx.stft = stft
        ctx.save_for_backward(y)
        return stft._forward(y)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_mel):
        (y,) = ctx.saved_tensors
        return None, ctx.stft.get_mel_backward(y, grad_mel)
