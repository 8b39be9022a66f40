"""Float64 numpy restatement of the mel front end's backward (csrc/mel.cu mel_bwd_kernel): the gradient of
log(clamp(basis @ |rfft(w * frame(pad(y)))|, clip)) with respect to y, written step by step from the math, not from
autograd.  Ground truth for tests/test_oracle_mel_grad.py, tests/test_emu_mel_backward.py and the GPU tests.

The weights are the float32 ones every implementation uses (librosa's filterbank, torch.hann_window), promoted to
float64, so only the arithmetic differs.  ``active`` overrides the clamp decision (a bool mask of the mel's shape)."""
import numpy as np
import torch

from oracle import mel as om

SR, N_MELS, N_FFT, FMIN, FMAX, CLIP = 44100, 128, 2048, 40, 16000, 1e-5


def tables():
    basis = om.librosa_mel(sr=SR, n_fft=N_FFT, n_mels=N_MELS, fmin=FMIN, fmax=FMAX).astype(np.float64)
    window = torch.hann_window(N_FFT).double().numpy()
    return basis, window


def padding(T, hop):
    """(src index of every padded position, valid mask): reflect, or constant when pad_right >= T (nvSTFT.py:97-103)"""
    pad_left = (N_FFT - hop) // 2
    pad_right = max((N_FFT - hop + 1) // 2, N_FFT - T - pad_left)
    idx = np.arange(-pad_left, T + pad_right)
    if pad_right < T:
        src = np.where(idx < 0, -idx, np.where(idx >= T, 2 * (T - 1) - idx, idx))
        return src, np.ones(idx.shape, bool)
    return np.clip(idx, 0, T - 1), (idx >= 0) & (idx < T)


def forward(y, hop):
    """float64 (Z [B, nF, 1025], mag, M [B, n_mels, nF], frame start indices, src, valid)"""
    y = np.asarray(y, np.float64)
    basis, window = tables()
    src, valid = padding(y.shape[1], hop)
    yp = y[:, src] * valid
    nF = 1 + (yp.shape[1] - N_FFT) // hop
    starts = hop * np.arange(nF)
    Z = np.fft.rfft(yp[:, starts[:, None] + np.arange(N_FFT)] * window, axis=-1)
    mag = np.sqrt(Z.real ** 2 + Z.imag ** 2 + 1e-9)
    M = np.einsum("mk,bfk->bmf", basis, mag)
    return Z, mag, M, starts, src, valid


def log_mel(y, hop):
    return np.log(np.maximum(forward(y, hop)[2], CLIP))


def mel_grad(y, hop, cot, active=None):
    """dL/dy [B, T] for L = sum(log_mel(y) * cot)"""
    y = np.asarray(y, np.float64)
    cot = np.asarray(cot, np.float64)
    B, T = y.shape
    basis, window = tables()
    Z, mag, M, starts, src, valid = forward(y, hop)
    if active is None:
        active = M >= CLIP                                    # torch's clamp(min=) passes the gradient at equality
    gM = np.where(active, cot / M, 0.0)                       # step 2
    gmag = np.einsum("mk,bmf->bfk", basis, gM)                # step 3: transposed projection
    G = gmag * Z / mag                                        # step 4: dL/dRe Z + j dL/dIm Z
    full = np.zeros(G.shape[:2] + (N_FFT,), complex)
    full[..., :N_FFT // 2 + 1] = G
    d = np.real(np.fft.ifft(full, axis=-1)) * N_FFT           # step 5: sum_{k<=1024} Re(G[k] e^{+2 pi i k n / N})
    dfr = d * window                                          # step 6
    dyp = np.zeros((B, src.shape[0]))
    for f, s in enumerate(starts):
        dyp[:, s:s + N_FFT] += dfr[:, f]
    out = np.zeros((B, T))                                    # step 7: fold the padding back
    for b in range(B):
        out[b] = np.bincount(src[valid], weights=dyp[b, valid], minlength=T)
    return out


def autograd64(y, hop, cot):
    """the reference's operators (oracle/mel.py, nvSTFT.py:97-115) under torch autograd in float64, on CPU"""
    import torch.nn.functional as F
    basis, window = tables()
    y = torch.as_tensor(np.asarray(y, np.float64)).requires_grad_(True)
    T = y.shape[-1]
    pad_left = (N_FFT - hop) // 2
    pad_right = max((N_FFT - hop + 1) // 2, N_FFT - T - pad_left)
    yp = F.pad(y.unsqueeze(1), (pad_left, pad_right), mode="reflect" if pad_right < T else "constant").squeeze(1)
    spec = torch.stft(yp, N_FFT, hop_length=hop, win_length=N_FFT, window=torch.from_numpy(window), center=False,
                      normalized=False, onesided=True, return_complex=True)
    spec = torch.sqrt(spec.real.pow(2) + spec.imag.pow(2) + 1e-9)
    mel = torch.log(torch.clamp(torch.matmul(torch.from_numpy(basis), spec), min=CLIP))
    (mel * torch.as_tensor(np.asarray(cot, np.float64))).sum().backward()
    return y.grad.numpy()
