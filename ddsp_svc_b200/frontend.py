"""Caller-side prologue / epilogue of the synthesis path on the GPU (SURVEY 8f rank 2): what the reference's inference
drivers do in numpy around `model(...)` -- Volume_Extractor (ddsp/vocoder.py:147-157), the silence mask (main.py:210-215),
`seg_output *= mask` (main.py:260) and the segment cross-fade (main.py:142-149) -- as streaming kernels of
libb200ddsp.so, so a rendered segment never has to leave the device between the synthesizer and the enhancer.
``slicer_rms`` and ``segment_place_`` are the two device halves of main.py's whole-file loop (offline.py): the Slicer's
frame RMS and the placement of one converted segment into the result.

``Volume_Extractor`` keeps the reference's constructor and ``extract`` contract (1-D numpy in -> 1-D numpy out) and
additionally accepts CUDA tensors ([T] or [B, T]) and then returns a CUDA tensor.
"""
import numpy as np
import torch

from . import _lib
from .ops import _count, _need_cuda_f32, _stream


def volume_extract(audio, hop_size):
    """audio [B, T] CUDA fp32 -> volume [B, T // hop + 1]."""
    _need_cuda_f32("audio", audio)
    if audio.dim() != 2:
        raise ValueError("audio must be [B, n_samples]")
    audio = audio.contiguous()
    B, T = audio.shape
    out = torch.empty(B, T // int(hop_size) + 1, dtype=torch.float32, device=audio.device)
    _lib.check(_lib.lib().b2d_volume_extract(audio.data_ptr(), B, T, int(hop_size), out.data_ptr(), _stream()), "b2d_volume_extract")
    _count(1)
    return out


def volume_mask(volume, threshold_db=-60.0):
    """volume [B, nF] -> mask [B, nF] in {0, 1}: (volume > 10**(dB/20)) dilated by 4 frames each side (main.py:211-213)."""
    _need_cuda_f32("volume", volume)
    if volume.dim() != 2:
        raise ValueError("volume must be [B, n_frames]")
    volume = volume.contiguous()
    B, nF = volume.shape
    out = torch.empty_like(volume)
    thr = mask_threshold(threshold_db)
    _lib.check(_lib.lib().b2d_volume_mask(volume.data_ptr(), B, nF, thr, out.data_ptr(), _stream()), "b2d_volume_mask")
    _count(1)
    return out


def mask_threshold(threshold_db):
    """the linear threshold volume_mask compares with: float32(10 ** (dB / 20))"""
    return float(np.float32(10 ** (float(threshold_db) / 20)))


def volume_mask_rows(volume, thresholds):
    """volume_mask with row b's linear threshold read from thresholds [B] (CUDA fp32, mask_threshold of each row's dB)
    when the kernel runs (b2d_volume_mask_rows)."""
    _need_cuda_f32("volume", volume)
    _need_cuda_f32("thresholds", thresholds)
    if volume.dim() != 2:
        raise ValueError("volume must be [B, n_frames]")
    volume = volume.contiguous()
    B, nF = volume.shape
    if thresholds.dim() != 1 or thresholds.numel() != B or not thresholds.is_contiguous():
        raise ValueError("thresholds must be a contiguous [%d] tensor, got %s" % (B, tuple(thresholds.shape)))
    out = torch.empty_like(volume)
    _lib.check(_lib.lib().b2d_volume_mask_rows(volume.data_ptr(), B, nF, thresholds.data_ptr(), out.data_ptr(),
                                               _stream()), "b2d_volume_mask_rows")
    _count(1)
    return out


def mask_apply_(signal, mask_frames, block_size, frame_offset=0):
    """In place: signal [B, n*block] *= upsample(mask_frames, block)[:, frame_offset*block : (frame_offset+n)*block]
    (main.py:215,260).  Returns ``signal``."""
    _need_cuda_f32("signal", signal)
    _need_cuda_f32("mask_frames", mask_frames)
    m = mask_frames.squeeze(-1) if mask_frames.dim() == 3 else mask_frames
    if signal.dim() != 2 or m.dim() != 2 or m.shape[0] != signal.shape[0] or not signal.is_contiguous():
        raise ValueError("signal must be contiguous [B, T] and mask_frames [B, n_frames(, 1)]")
    block = int(block_size)
    if signal.shape[1] % block != 0:
        raise ValueError("signal length %d is not a multiple of the block size %d" % (signal.shape[1], block))
    m = m.contiguous()
    n = signal.shape[1] // block
    _lib.check(_lib.lib().b2d_mask_apply(signal.data_ptr(), m.data_ptr(), signal.shape[0], m.shape[1], int(frame_offset), n,
                                         block, _stream()), "b2d_mask_apply")
    _count(1)
    return signal


def cross_fade(a, b, idx):
    """torch version of main.py:142-149 for 1-D CUDA fp32 tensors: -> tensor of idx + len(b) samples."""
    _need_cuda_f32("a", a)
    _need_cuda_f32("b", b)
    if a.dim() != 1 or b.dim() != 1:
        raise ValueError("cross_fade takes 1-D tensors")
    a, b = a.contiguous(), b.contiguous()
    out = torch.empty(int(idx) + b.shape[0], dtype=torch.float32, device=a.device)
    _lib.check(_lib.lib().b2d_cross_fade(a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], int(idx), out.data_ptr(), _stream()),
               "b2d_cross_fade")
    _count(1)
    return out


def slicer_rms_frames(n_samples, frame_length, hop):
    """the frames librosa.feature.rms(center=True) makes of n_samples: 1 + (n + 2 (frame_length // 2) - frame_length) // hop"""
    return 1 + (int(n_samples) + 2 * (int(frame_length) // 2) - int(frame_length)) // int(hop)


def slicer_rms(audio, frame_length, hop):
    """audio [N] CUDA fp32 -> rms [slicer_rms_frames(N, frame_length, hop)]: librosa.feature.rms(y=audio,
    frame_length=frame_length, hop_length=hop) as the reference's Slicer calls it (center=True, zero padding), in fp64
    rounded to fp32 (b2d_slicer_rms)."""
    _need_cuda_f32("audio", audio)
    if audio.dim() != 1:
        raise ValueError("audio must be 1-D [n_samples]")
    audio = audio.contiguous()
    out = torch.empty(slicer_rms_frames(audio.shape[0], frame_length, hop), dtype=torch.float32, device=audio.device)
    _lib.check(_lib.lib().b2d_slicer_rms(audio.data_ptr(), audio.shape[0], int(frame_length), int(hop), out.data_ptr(),
                                         _stream()), "b2d_slicer_rms")
    _count(1)
    return out


def segment_place_(result, seg, idx, fade_len):
    """In place: result[idx : idx + len(seg)] = seg, its first fade_len samples cross-faded against what result holds
    there with numpy.linspace(0, 1, fade_len) in fp64 (main.py:142-149 and :266-273; b2d_segment_place).  Returns
    ``result``."""
    _need_cuda_f32("result", result)
    _need_cuda_f32("seg", seg)
    if result.dim() != 1 or seg.dim() != 1 or not result.is_contiguous():
        raise ValueError("segment_place_ takes a contiguous 1-D result and a 1-D segment")
    seg = seg.contiguous()
    _lib.check(_lib.lib().b2d_segment_place(result.data_ptr(), result.shape[0], seg.data_ptr(), seg.shape[0], int(idx),
                                            int(fade_len), _stream()), "b2d_segment_place")
    _count(1)
    return result


class Volume_Extractor:
    """Drop-in for ddsp.vocoder.Volume_Extractor (ddsp/vocoder.py:147-157) running on the GPU."""

    def __init__(self, hop_size=512, device=None):
        self.hop_size = hop_size
        self.device = device

    def extract(self, audio):
        if isinstance(audio, np.ndarray):           # the reference's contract: 1-D numpy in, 1-D numpy out
            dev = self.device or "cuda"
            x = torch.from_numpy(np.ascontiguousarray(audio, dtype=np.float32)).to(dev).reshape(1, -1)
            return volume_extract(x, self.hop_size)[0].cpu().numpy().astype(audio.dtype if audio.dtype.kind == "f" else np.float32)
        if audio.dim() == 1:
            return volume_extract(audio.reshape(1, -1), self.hop_size)[0]
        return volume_extract(audio, self.hop_size)
