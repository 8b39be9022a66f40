"""gui.py's real-time conversion block (audio_callback, gui.py:393-460, with SvcDDSP.infer, gui.py:75-148) on the
device, replayed as CUDA graphs.

``RealtimeVC(model_path, samplerate, block_time, crossfade_time, extra_time, f0_min, f0_max, threhold, spk_id,
pitch_adjust, use_spk_mix, spk_mix_dict, use_enhancer, enhancer_adaptive_key, use_phase_vocoder, graph=True)`` takes
the fields of gui.py's Config and builds SvcDDSP's models from the package's classes.  ``process(indata [frames,
channels]) -> outdata [frames, 2]`` is one callback.

Per call: one host-to-device copy of the new block into the device ring buffer, then

- graph A: RMVPE -> rt_f0_regrid (F0_Extractor's post-processing and the pitch factor) -> volume -> mask -> units ->
  synthesizer -> mask multiply -> max f0 (for the 'auto' key);
- graph B[key]: enhancer -> resampling to the device rate -> rt_sola -> rt_crossfade -> copy to a pinned buffer.

With ``enhancer_adaptive_key='auto'`` the one read mid-block is the 4-byte max f0 between A and B; the other
synchronisation is the output copy.  One B graph is captured, on first use, per adaptive key.  The synthesizer's and
the enhancer's noise is drawn with torch's CUDA generator into static buffers (torch advances its graph-safe RNG on
every replay), not by the in-kernel Philox, whose seed is a host integer and would be frozen at capture.  Everything
host-derived is built before capture.  The session captures and replays on a stream it owns, so ``process`` may be
called from the sounddevice callback thread.  ``graph=False`` runs the same code eagerly.
"""
import numpy as np
import torch

from . import frontend, ops
from .dropin import load_model
from .enhancer import Enhancer, adaptive_rate, auto_key
from .hubert import Units_Encoder
from .rmvpe import RMVPE, Resampler

# the largest f0 RMVPE decodes (cents 20 * 359 + 1997.38 above 10 Hz): bounds the keys 'auto' can pick
RMVPE_F0_MAX = 10 * 2 ** ((20 * 359 + 1997.3794084376191) / 1200)


class RealtimeVC:
    def __init__(self, model_path, samplerate=44100, block_time=0.3, crossfade_time=0.04, extra_time=2.0, f0_min=50,
                 f0_max=1100, threhold=-45, spk_id=1, pitch_adjust=0.0, use_spk_mix=False, spk_mix_dict=None,
                 use_enhancer=True, enhancer_adaptive_key=0, use_phase_vocoder=False, graph=True,
                 pitch_extractor_type="rmvpe", rmvpe_ckpt="pretrain/rmvpe/model.pt", device=None):
        if pitch_extractor_type != "rmvpe":
            raise ValueError("RealtimeVC extracts f0 with 'rmvpe' only: %r has no kernels" % (pitch_extractor_type,))
        self.device = torch.device("cuda" if device is None else device)
        if self.device.type != "cuda":
            raise ValueError("RealtimeVC runs on the CUDA kernels: device must be a CUDA device")
        self.sr = int(samplerate)
        self.block = int(block_time * self.sr)
        self.cf = int(crossfade_time * self.sr)
        self.search = int(0.01 * self.sr)
        self.delay = int(0.02 * self.sr)
        extra = int(extra_time * self.sr)
        self.n_in = max(self.block + self.cf + self.search + 2 * self.delay, self.block + extra)
        pad = extra_time - crossfade_time - 0.01 - 0.02                 # f_safe_prefix_pad_length
        self.silence_front = pad - 0.03 if pad > 0.03 else 0
        self.f0_min, self.f0_max = float(f0_min), float(f0_max)
        self.pitch_adjust = float(pitch_adjust)
        self.pitch_factor = 2 ** (self.pitch_adjust / 12)
        self.threhold = float(threhold)
        self.use_enhancer, self.key = bool(use_enhancer), enhancer_adaptive_key
        self.use_pv, self.graph = bool(use_phase_vocoder), bool(graph)

        self.model, self.args = load_model(model_path, device=self.device)
        data = self.args.data
        self.model_sr, self.block_size = int(data.sampling_rate), int(data.block_size)
        hop = self.block_size * self.sr / self.model_sr
        if hop != int(hop):
            raise ValueError("the hop at %d Hz is %g samples: RealtimeVC's volume kernel needs an integer hop "
                             "(block_size * samplerate / model sampling_rate)" % (self.sr, hop))
        self.hop = int(hop)
        self.units_encoder = Units_Encoder(data.encoder, data.encoder_ckpt, data.encoder_sample_rate,
                                           data.encoder_hop_size, device=self.device,
                                           cnhubertsoft_gate=getattr(data, "cnhubertsoft_gate", None) or 10)
        self.rmvpe = RMVPE(rmvpe_ckpt, hop_length=160)
        self.enhancer = Enhancer(self.args.enhancer.type, self.args.enhancer.ckpt, self.device) if use_enhancer else None
        self.out_sr = self.enhancer.enhancer_sample_rate if use_enhancer else self.model_sr
        self.to_device_rate = Resampler(self.sr)

        dev = self.device
        self.n_frames = self.n_in // self.hop + 1
        self.start_frame = int(self.silence_front * self.sr / self.hop)
        self.trim = int(np.round(self.start_frame * self.hop / self.sr * self.sr))
        self.spk_id = torch.LongTensor(np.array([[spk_id]])).to(dev)
        self.spk_mix_dict = spk_mix_dict if use_spk_mix else None
        self.ring = torch.zeros(self.n_in, device=dev)
        self.new_block = torch.zeros(self.block, device=dev)
        self.sola_buffer = torch.zeros(self.cf, device=dev)
        self.fade_in = torch.sin(np.pi * torch.arange(0, 1, 1 / self.cf, device=dev) / 2) ** 2
        self.fade_out = 1 - self.fade_in
        # the synthesizer's noise: randn for CombSubSuperFast, uniform in [-1, 1) for the others (ddsp/vocoder.py)
        self.noise = torch.zeros(1, self.n_frames * self.block_size, device=dev)
        self.noise_normal = self.args.model.type == "CombSubSuperFast"
        if use_enhancer:
            ehop = self.enhancer.enhancer_hop_size
            top = adaptive_rate(self.enhancer.enhancer_sample_rate, self.max_key())[0]
            n_mel = int(self.noise.shape[1] * top / self.model_sr) // ehop + 4
            self.gen_rand_ini = torch.zeros(1, 1, 9, device=dev)
            self.gen_noise = torch.zeros(1, n_mel * ehop, 9, device=dev)
            self.enhancer.prepare(self.model_sr, [self.key] if self.key != "auto" else range(self.max_key() + 1))
        self.in_host = torch.zeros(self.block, dtype=torch.float32).pin_memory()
        self.out_host = torch.zeros(self.block, dtype=torch.float32).pin_memory()
        self.ratio_host = torch.zeros(1, dtype=torch.float32).pin_memory()
        self.stream = torch.cuda.Stream(device=dev)
        self.graph_a, self.graphs_b = None, {}

    def max_key(self):
        """the largest adaptive key 'auto' can pick for the f0 RMVPE decodes, after the pitch factor"""
        return int(auto_key(max(RMVPE_F0_MAX, self.f0_min) * self.pitch_factor / 760))

    def _draw_noise(self):
        if self.noise_normal:
            self.noise.normal_()
        else:
            self.noise.uniform_(-1, 1)

    def _draw_enhancer_noise(self):
        self.gen_rand_ini.uniform_()                                    # SineGen's rand_ini: torch.rand, first zero
        self.gen_rand_ini[..., 0] = 0
        self.gen_noise.normal_()

    # ---- the two halves of the block ----------------------------------------------------------------------------------
    def _stage_a(self):
        """ring buffer -> masked synthesizer output [1, T] and max(f0[start_frame:]) / 760"""
        self.ring.copy_(torch.cat([self.ring[self.block:], self.new_block]))
        audio = self.ring[None]
        f0_10ms = self.rmvpe.infer_batch(audio[:, self.trim:], self.sr)[0]
        f0 = ops.rt_f0_regrid(f0_10ms.contiguous(), 0.01, self.n_frames, self.hop / self.sr, rmvpe=True,
                              pad=self.start_frame, f0_min=self.f0_min, post_scale=self.pitch_factor)
        f0 = f0[None, :, None]
        volume = frontend.volume_extract(audio, self.hop)
        mask = frontend.volume_mask(volume, self.threhold)
        units = self.units_encoder.encode(audio, self.sr, self.hop)
        self._draw_noise()
        with torch.no_grad():
            out, _, _ = self.model(units, f0, volume[..., None], spk_id=self.spk_id, spk_mix_dict=self.spk_mix_dict,
                                   noise=self.noise)
        out = frontend.mask_apply_(out.contiguous(), mask, self.block_size)
        ratio = torch.max(f0[:, self.start_frame:]) / 760
        return out, f0, ratio

    def _stage_b(self, out, f0, key):
        """synthesizer output -> the block in the pinned output buffer; the SOLA buffer advanced"""
        if self.use_enhancer:
            self._draw_enhancer_noise()
            out, _ = self.enhancer.enhance(out, self.model_sr, f0, self.block_size, adaptive_key=key,
                                           silence_front=self.silence_front, rand_ini=self.gen_rand_ini,
                                           noise=self.gen_noise)
        audio = out.reshape(1, -1)
        if self.out_sr != self.sr:
            audio = self.to_device_rate(audio.contiguous(), self.out_sr)
        audio = audio[0]
        temp = audio[audio.numel() - self.block - self.cf - self.search - self.delay:audio.numel() - self.delay]
        shift = ops.rt_sola(temp, self.sola_buffer, self.search)
        block_out, nxt = ops.rt_crossfade(temp, shift, self.search, self.sola_buffer, self.fade_in, self.fade_out,
                                          self.block, self.use_pv)
        self.sola_buffer.copy_(nxt)
        self.out_host.copy_(block_out, non_blocking=True)

    def _capture(self, fn, state):
        """fn captured on the session's stream after one eager warm-up run (tables, packed weights, allocator); the
        warm-up's writes to the session state tensors are undone, so the first replay starts where it should"""
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            saved = [t.clone() for t in state]
            fn()
            for t, v in zip(state, saved):
                t.copy_(v)
        self.stream.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=self.stream):
            static = fn()
        return g, static

    # ---- one callback -------------------------------------------------------------------------------------------------
    def upload(self, indata):
        """the new block (mono as librosa.to_mono averages channels) into the device staging buffer"""
        x = np.asarray(indata, dtype=np.float32)
        mono = x.mean(axis=1, dtype=np.float32) if x.ndim == 2 and x.shape[1] > 1 else x.reshape(-1)
        if mono.shape[0] != self.block:
            raise ValueError("indata holds %d frames; the session's block is %d" % (mono.shape[0], self.block))
        self.in_host.numpy()[:] = mono
        with torch.cuda.stream(self.stream):
            self.new_block.copy_(self.in_host, non_blocking=True)

    def run_a(self):
        """enqueue graph A (or its eager code) on the session's stream"""
        if not self.graph:
            with torch.cuda.stream(self.stream):
                self._a = self._stage_a()
        else:
            if self.graph_a is None:
                self.graph_a, self._a = self._capture(self._stage_a, [self.ring])
            with torch.cuda.stream(self.stream):                        # a replay runs on the current stream
                self.graph_a.replay()

    def pick_key(self):
        """the adaptive key of this block; with 'auto', reads max f0 from the device (the block's one mid-block sync)"""
        if self.key != "auto":
            return float(self.key)
        with torch.cuda.stream(self.stream):
            self.ratio_host.copy_(self._a[2].reshape(1), non_blocking=True)
        self.stream.synchronize()
        return float(auto_key(float(self.ratio_host[0])))

    def run_b(self, key):
        """enqueue graph B[key] (or its eager code) on the session's stream"""
        out, f0, _ = self._a
        if not self.graph:
            with torch.cuda.stream(self.stream):
                self._stage_b(out, f0, key)
            return
        g = self.graphs_b.get(key)
        if g is None:
            if self.use_enhancer:
                self.enhancer.prepare(self.model_sr, [key])
            g, _ = self._capture(lambda: self._stage_b(out, f0, key), [self.sola_buffer])
            self.graphs_b[key] = g
        with torch.cuda.stream(self.stream):
            g.replay()

    def process(self, indata):
        """audio_callback's math: indata [frames, channels] -> outdata [frames, 2] (float32)"""
        self.upload(indata)
        self.run_a()
        self.run_b(self.pick_key())
        self.stream.synchronize()
        return np.repeat(self.out_host.numpy()[:, None], 2, axis=1)
