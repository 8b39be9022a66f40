"""Drop-in for the reference's ``Enhancer`` (enhancer.py:8-85): the NSF-HiFiGAN enhancer that main.py and gui.py run
on the DDSP output, on the kernels end to end.

``Enhancer(enhancer_type, enhancer_ckpt, device=None)`` loads the package's ``Generator`` from the checkpoint and its
config.json.  ``enhance(audio [B, T], sample_rate, f0 [B, n_frames, 1], hop_size, adaptive_key=0, silence_front=0)
-> (audio [B, 1, T'], enhancer_sample_rate)`` keeps the reference's contract:

- audio is resampled to the adaptive rate and back with torchaudio's lowpass_filter_width=128 table
  (rmvpe.Resampler), on the kernels;
- f0 is regridded on the device by ``ops.rt_f0_regrid`` (np.interp in fp64, scaled by real_factor, held at the
  edges), so a numeric ``adaptive_key`` reads nothing back from the device; ``'auto'`` reads one scalar, as the
  reference's ``float(torch.max(f0))`` does, and prints the key it picked as the reference does;
- the mel is ``mel.STFT.get_mel`` at keyshift 0 and the vocoder the package's ``Generator``.

Two additions serve graph capture (realtime.RealtimeVC): ``prepare(sample_rate, keys)`` builds the resampling tables
of those adaptive keys ahead of time, and ``enhance(..., rand_ini=, noise=)`` takes the generator's draws from the
caller ([1, 1, 9] and [B, >= n_mel_frames hop, 9]) instead of the in-kernel generator, whose seed is a host integer.
A third serves independent sessions in one batch (realtime.BatchedRealtimeVC): audio [B, T] and f0 [B, n_frames, 1]
at a numeric key, every row enhanced on its own; 'auto' would pick one key per row, so it takes B = 1.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import ops
from .mel import STFT
from .nsf_vocoder import load_generator
from .rmvpe import Resampler


def adaptive_rate(enhancer_sample_rate, adaptive_key):
    """Enhancer.enhance's adaptive sample rate and real_factor for a numeric key"""
    factor = 2 ** (-float(adaptive_key) / 12)
    rate = 100 * int(np.round(enhancer_sample_rate / factor / 100))
    return rate, enhancer_sample_rate / rate


def auto_key(ratio):
    """the key 'auto' picks for ratio = max(f0) / 760 (fp32 on the device, as the reference divides it)"""
    return max(0, np.ceil(12 * np.log2(ratio)))


class Enhancer:
    def __init__(self, enhancer_type, enhancer_ckpt, device=None):
        if enhancer_type != "nsf-hifigan":
            raise ValueError(f" [x] Unknown enhancer: {enhancer_type}")
        device = torch.device("cuda" if device is None else device)
        if device.type != "cuda":
            raise ValueError("the enhancer runs on the CUDA kernels: device must be a CUDA device, got %s" % device)
        self.device = device
        print('| Load HifiGAN: ', enhancer_ckpt)
        self.model, self.h = load_generator(enhancer_ckpt, device)
        h = self.h
        self.stft = STFT(h.sampling_rate, h.num_mels, h.n_fft, h.win_size, h.hop_size, h.fmin, h.fmax)
        self.enhancer_sample_rate = h.sampling_rate
        self.enhancer_hop_size = h.hop_size
        self.resample_kernel = {}                           # target rate -> rmvpe.Resampler (its tables by source rate)

    def _resampler(self, new_freq):
        if new_freq not in self.resample_kernel:
            self.resample_kernel[new_freq] = Resampler(new_freq)
        return self.resample_kernel[new_freq]

    def _resample(self, audio, orig_freq, new_freq):
        return self._resampler(new_freq)(audio.float().contiguous(), orig_freq)

    def prepare(self, sample_rate, keys):
        """build the resampling tables enhance() needs at these numeric adaptive keys for audio at sample_rate"""
        x = torch.zeros(1, 4096, device=self.device)
        for key in keys:
            rate, _ = adaptive_rate(self.enhancer_sample_rate, key)
            if rate != sample_rate:
                self._resampler(rate)(x, sample_rate)
            if rate != self.enhancer_sample_rate:
                self._resampler(self.enhancer_sample_rate)(x, rate)

    def enhance(self, audio, sample_rate, f0, hop_size, adaptive_key=0, silence_front=0, rand_ini=None, noise=None):
        if not (isinstance(audio, torch.Tensor) and audio.is_cuda and audio.dim() == 2):
            raise ValueError("audio must be a [B, T] CUDA tensor")
        B = audio.shape[0]
        if not (isinstance(f0, torch.Tensor) and f0.is_cuda and f0.dim() == 3 and f0.shape[0] == B):
            raise ValueError("f0 must be a [B, n_frames, 1] CUDA tensor with audio's B = %d rows" % B)
        if adaptive_key == 'auto' and B != 1:
            raise ValueError("adaptive_key 'auto' picks a key, and so a sample rate, from one utterance's f0: enhance "
                             "%d rows at a numeric key, or one row at a time" % B)
        start_frame = int(silence_front * sample_rate / hop_size)
        real_silence_front = start_frame * hop_size / sample_rate
        audio = audio[:, int(np.round(real_silence_front * sample_rate)):]
        f0 = f0[:, start_frame:, :]
        if adaptive_key == 'auto':
            adaptive_key = auto_key(float(torch.max(f0) / 760))
            print('auto_adaptive_key: ' + str(int(adaptive_key)))
        rate, real_factor = adaptive_rate(self.enhancer_sample_rate, adaptive_key)
        audio_res = audio if sample_rate == rate else self._resample(audio, sample_rate, rate)
        n_frames = int(audio_res.size(-1) // self.enhancer_hop_size + 1)
        if hop_size == self.enhancer_hop_size and sample_rate == self.enhancer_sample_rate and sample_rate == rate:
            f0_res = f0.squeeze(-1)
        else:
            f0_res = ops.rt_f0_regrid_batch(f0[:, :, 0].float().contiguous(), hop_size / sample_rate, n_frames,
                                            self.enhancer_hop_size / self.enhancer_sample_rate, src_div=real_factor,
                                            src_scale=real_factor)
        with torch.no_grad():
            mel = self.stft.get_mel(audio_res)
            if noise is not None:
                noise = noise[:, :mel.size(-1) * self.enhancer_hop_size]
            enhanced = self.model(mel, f0_res[:, :mel.size(-1)], rand_ini=rand_ini, noise=noise)
        if rate != self.enhancer_sample_rate:
            enhanced = self._resample(enhanced.reshape(B, -1), rate, self.enhancer_sample_rate).unsqueeze(1)
        if start_frame > 0:
            enhanced = F.pad(enhanced, (int(np.round(self.enhancer_sample_rate * real_silence_front)), 0))
        return enhanced, self.enhancer_sample_rate
