"""The key-shifted mel (nvSTFT.py:73-117 with keyshift != 0, speed 1, center False) restated for the tests and
bench_keyshift_mel.py: in float64 (the accuracy reference), and in fp32 eagerly with its tables already on the input's
device (the reference's algorithm on torch.stft / cuFFT, what the kernel is timed against)."""
import torch
import torch.nn.functional as F

from oracle import mel as om


def n_fft_new(keyshift, n_fft=2048):
    import numpy as np
    return int(np.round(n_fft * 2 ** (keyshift / 12)))


def basis(dtype=torch.float32, device="cpu"):
    return torch.from_numpy(om.librosa_mel(44100, 2048, 128, 40, 16000)).to(device=device, dtype=dtype)


def get_mel(y, hop, keyshift, mel_basis=None, window=None, clip_val=1e-5):
    """y [B, T] in its own dtype and device -> [B, 128, n_frames].  mel_basis / window: the 2048-point filterbank and
    hann(n') on y's device (built when None)"""
    n = n_fft_new(keyshift)
    mel_basis = basis(y.dtype, y.device) if mel_basis is None else mel_basis
    window = torch.hann_window(n, dtype=y.dtype, device=y.device) if window is None else window
    T = y.size(-1)
    pad_left = (n - hop) // 2
    pad_right = max((n - hop + 1) // 2, n - T - pad_left)
    y = F.pad(y.unsqueeze(1), (pad_left, pad_right), mode="reflect" if pad_right < T else "constant").squeeze(1)
    s = torch.stft(y, n, hop_length=hop, win_length=n, window=window, center=False, return_complex=True)
    s = torch.sqrt(s.real.pow(2) + s.imag.pow(2) + 1e-9)
    if s.size(1) < 1025:
        s = F.pad(s, (0, 0, 0, 1025 - s.size(1)))
    s = s[:, :1025, :] * 2048 / n
    return torch.log(torch.clamp(torch.matmul(mel_basis, s), min=clip_val))


def mel64(y, hop, keyshift):
    """get_mel in float64 (the fp32 filterbank values, exactly)"""
    return get_mel(y.double(), hop, keyshift)
