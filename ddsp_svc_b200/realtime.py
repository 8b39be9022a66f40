"""The real-time conversion blocks of gui.py and gui_reflow.py on the device, replayed as CUDA graphs.

``RealtimeVC(model_path, samplerate, block_time, crossfade_time, extra_time, f0_min, f0_max, threhold, spk_id,
pitch_adjust, use_spk_mix, spk_mix_dict, use_enhancer, enhancer_adaptive_key, use_phase_vocoder, graph=True)`` takes
the fields of gui.py's Config and builds SvcDDSP's models from the package's classes (audio_callback, gui.py:393-460,
with SvcDDSP.infer, gui.py:75-148).  ``process(indata [frames, channels]) -> outdata [frames, 2]`` is one callback.

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

``RealtimeReflowVC(model_path, ..., formant_shift_key, t_start, infer_step, sampling_method, ...)`` is gui_reflow.py's
block (audio_callback, gui_reflow.py:421-489, with SvcDDSP.infer, :66-151) on the reflow model's cascade
(reflow_vocoder.Unit2Wav): ring buffer -> RMVPE -> rt_f0_regrid -> volume -> mask -> units -> CombSubSuperFast with the
formant key as aug_shift -> mel -> rectified-flow sampler -> NSF-HiFiGAN -> mask multiply -> resampling -> rt_sola ->
rt_crossfade -> pinned copy, ONE graph: no value in it is data-dependent.  Its draws (the DDSP noise, the sampler's
initial noise, SineGen's rand_ini and noise) are static buffers filled by torch's CUDA generator, and the sampler's step
rows are cached by RectifiedFlow after the warm-up, so a replay copies nothing to the device and never synchronises.

Both sessions share ``_Session``: the ring buffer, the upload and the owned stream, capture with a warm-up and a state
restore, the f0 / volume / mask / units front half, the resampling -> SOLA -> crossfade -> pinned-copy tail and
SineGen's draws.  ``reflow_frames`` is the reflow block's frame bookkeeping as a pure function.
"""
import numpy as np
import torch

from . import frontend, ops
from .dropin import load_model
from .enhancer import Enhancer, adaptive_rate, auto_key
from .hubert import Units_Encoder
from .reflow_vocoder import load_model_vocoder
from .rmvpe import RMVPE, Resampler, resampled_length

# the largest f0 RMVPE decodes (cents 20 * 359 + 1997.38 above 10 Hz): bounds the keys 'auto' can pick
RMVPE_F0_MAX = 10 * 2 ** ((20 * 359 + 1997.3794084376191) / 1200)
SINEGEN_DIM = 9                                                         # NSF-HiFiGAN's SineGen: harmonic_num 8


def gui_frames(samplerate, block_time, crossfade_time, extra_time):
    """GUI.set_values of gui.py / gui_reflow.py: block, crossfade, SOLA search, delay and input lengths in samples, and
    SvcDDSP.infer's silence_front in seconds (from f_safe_prefix_pad_length)"""
    sr = int(samplerate)
    block, cf = int(block_time * sr), int(crossfade_time * sr)
    search, delay, extra = int(0.01 * sr), int(0.02 * sr), int(extra_time * sr)
    pad = extra_time - crossfade_time - 0.01 - 0.02
    return dict(sr=sr, block=block, cf=cf, search=search, delay=delay,
                n_in=max(block + cf + search + 2 * delay, block + extra), silence_front=pad - 0.03 if pad > 0.03 else 0)


def model_hop(samplerate, model_sr, block_size, who):
    """block_size * samplerate / model sampling_rate: the frame hop at the device rate, which must be an integer"""
    hop = block_size * samplerate / model_sr
    if hop != int(hop):
        raise ValueError("the hop at %d Hz is %g samples: %s's volume kernel needs an integer hop "
                         "(block_size * samplerate / model sampling_rate)" % (samplerate, hop, who))
    return int(hop)


def reflow_frames(samplerate, block_time, crossfade_time, extra_time, model_sr, block_size, vocoder_hop,
                  win_size=2048):
    """The frame bookkeeping of one gui_reflow.py block -> dict:

    - gui_frames' lengths and silence_front; ``hop`` and ``n_frames`` (F0_Extractor's and the volume's frames);
    - ``start_frame`` / ``trim``: F0_Extractor's leading frames and the samples RMVPE skips;
    - ``mel_start``: Unit2Wav's start_frame, from the model rate; ``mel_frames``: the mel of the DDSP output from there
      (nvSTFT's padding, center=False); ``out_len``: the vocoder's samples at the model rate;
    - ``mask_offset``: the mask frame ``mask[:, -output.shape[-1]:]`` starts at;
    - ``out_dev``: the output's length at the device rate, and ``tail``: the (start, stop) of the samples SOLA reads.
    The output always covers the SOLA window: silence_front leaves crossfade_time + 0.06 s of the ring before the block.
    Raises ValueError where the block cannot run: a non-integer hop, or an output that is not whole mask frames."""
    f = gui_frames(samplerate, block_time, crossfade_time, extra_time)
    sr = f["sr"]
    hop = model_hop(sr, model_sr, block_size, "RealtimeReflowVC")
    n_frames = f["n_in"] // hop + 1
    start_frame = int(f["silence_front"] * sr / hop)
    mel_start = int(f["silence_front"] * model_sr / block_size)
    n = (n_frames - mel_start) * block_size
    pad_left = (win_size - vocoder_hop) // 2
    pad_right = max((win_size - vocoder_hop + 1) // 2, win_size - n - pad_left)
    mel_frames = (n + pad_left + pad_right - win_size) // vocoder_hop + 1
    out_len = mel_frames * vocoder_hop
    if out_len % block_size or out_len > n_frames * block_size:
        raise ValueError("the vocoder's %d samples are not whole frames of the %d-sample mask" % (out_len, block_size))
    out_dev = out_len if model_sr == sr else resampled_length(out_len, model_sr, sr)
    tail = (out_dev - f["block"] - f["cf"] - f["search"] - f["delay"], out_dev - f["delay"])
    f.update(hop=hop, n_frames=n_frames, start_frame=start_frame,
             trim=int(np.round(start_frame * hop / sr * sr)), mel_start=mel_start, mel_frames=mel_frames,
             out_len=out_len, mask_offset=n_frames - out_len // block_size, out_dev=out_dev, tail=tail)
    return f


class _Session:
    """What the gui.py and gui_reflow.py sessions share (see the module's docstring)"""

    def _init_block(self, samplerate, block_time, crossfade_time, extra_time, device, who):
        self.device = torch.device("cuda" if device is None else device)
        if self.device.type != "cuda":
            raise ValueError("%s runs on the CUDA kernels: device must be a CUDA device" % who)
        f = gui_frames(samplerate, block_time, crossfade_time, extra_time)
        self.sr, self.block, self.cf, self.search, self.delay = f["sr"], f["block"], f["cf"], f["search"], f["delay"]
        self.n_in, self.silence_front = f["n_in"], f["silence_front"]

    def _init_front(self, data, f0_min, threhold, pitch_adjust, spk_id, use_spk_mix, spk_mix_dict, rmvpe_ckpt, who):
        """the f0 / volume / mask / units half (models, frames, ring and staging buffers) and the SOLA state; ``data``:
        the checkpoint config's data section"""
        dev = self.device
        self.f0_min = float(f0_min)
        self.pitch_adjust = float(pitch_adjust)
        self.pitch_factor = 2 ** (self.pitch_adjust / 12)
        self.threhold = float(threhold)
        self.model_sr, self.block_size = int(data.sampling_rate), int(data.block_size)
        self.hop = model_hop(self.sr, self.model_sr, self.block_size, who)
        self.units_encoder = Units_Encoder(data.encoder, data.encoder_ckpt, data.encoder_sample_rate,
                                           data.encoder_hop_size, device=dev,
                                           cnhubertsoft_gate=getattr(data, "cnhubertsoft_gate", None) or 10)
        self.rmvpe = RMVPE(rmvpe_ckpt, hop_length=160)
        self.to_device_rate = Resampler(self.sr)
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
        self.in_host = torch.zeros(self.block, dtype=torch.float32).pin_memory()
        self.out_host = torch.zeros(self.block, dtype=torch.float32).pin_memory()
        self.stream = torch.cuda.Stream(device=dev)

    @staticmethod
    def _draw_sinegen(rand_ini, noise):
        """SineGen's draws into static buffers: rand_ini torch.rand with its first entry zeroed, noise randn"""
        rand_ini.uniform_()
        rand_ini[..., 0] = 0
        noise.normal_()

    def _front(self):
        """ring buffer -> f0 [1, n_frames, 1] (pitch factor applied), volume [1, n_frames], mask [1, n_frames], units"""
        self.ring.copy_(torch.cat([self.ring[self.block:], self.new_block]))
        audio = self.ring[None]
        f0_10ms = self.rmvpe.infer_batch(audio[:, self.trim:], self.sr)[0]
        f0 = ops.rt_f0_regrid(f0_10ms.contiguous(), 0.01, self.n_frames, self.hop / self.sr, rmvpe=True,
                              pad=self.start_frame, f0_min=self.f0_min, post_scale=self.pitch_factor)
        f0 = f0[None, :, None]
        volume = frontend.volume_extract(audio, self.hop)
        mask = frontend.volume_mask(volume, self.threhold)
        units = self.units_encoder.encode(audio, self.sr, self.hop)
        return f0, volume, mask, units

    def _tail(self, out, out_sr):
        """audio [1, T] at out_sr -> the block in the pinned output buffer; the SOLA buffer advanced"""
        audio = out.reshape(1, -1)
        if out_sr != self.sr:
            audio = self.to_device_rate(audio.contiguous(), out_sr)
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

    def upload(self, indata):
        """the new block (mono as librosa.to_mono averages channels) into the device staging buffer"""
        x = np.asarray(indata, dtype=np.float32)
        mono = x.mean(axis=1, dtype=np.float32) if x.ndim == 2 and x.shape[1] > 1 else x.reshape(-1)
        if mono.shape[0] != self.block:
            raise ValueError("indata holds %d frames; the session's block is %d" % (mono.shape[0], self.block))
        self.in_host.numpy()[:] = mono
        with torch.cuda.stream(self.stream):
            self.new_block.copy_(self.in_host, non_blocking=True)

    def _output(self):
        self.stream.synchronize()
        return np.repeat(self.out_host.numpy()[:, None], 2, axis=1)


class RealtimeVC(_Session):
    def __init__(self, model_path, samplerate=44100, block_time=0.3, crossfade_time=0.04, extra_time=2.0, f0_min=50,
                 f0_max=1100, threhold=-45, spk_id=1, pitch_adjust=0.0, use_spk_mix=False, spk_mix_dict=None,
                 use_enhancer=True, enhancer_adaptive_key=0, use_phase_vocoder=False, graph=True,
                 pitch_extractor_type="rmvpe", rmvpe_ckpt="pretrain/rmvpe/model.pt", device=None):
        if pitch_extractor_type != "rmvpe":
            raise ValueError("RealtimeVC extracts f0 with 'rmvpe' only: %r has no kernels" % (pitch_extractor_type,))
        self._init_block(samplerate, block_time, crossfade_time, extra_time, device, "RealtimeVC")
        self.f0_max = float(f0_max)
        self.use_enhancer, self.key = bool(use_enhancer), enhancer_adaptive_key
        self.use_pv, self.graph = bool(use_phase_vocoder), bool(graph)

        self.model, self.args = load_model(model_path, device=self.device)
        self._init_front(self.args.data, f0_min, threhold, pitch_adjust, spk_id, use_spk_mix, spk_mix_dict,
                         rmvpe_ckpt, "RealtimeVC")
        self.enhancer = Enhancer(self.args.enhancer.type, self.args.enhancer.ckpt, self.device) if use_enhancer else None
        self.out_sr = self.enhancer.enhancer_sample_rate if use_enhancer else self.model_sr

        dev = self.device
        # the synthesizer's noise: randn for CombSubSuperFast, uniform in [-1, 1) for the others (ddsp/vocoder.py)
        self.noise = torch.zeros(1, self.n_frames * self.block_size, device=dev)
        self.noise_normal = self.args.model.type == "CombSubSuperFast"
        if use_enhancer:
            ehop = self.enhancer.enhancer_hop_size
            top = adaptive_rate(self.enhancer.enhancer_sample_rate, self.max_key())[0]
            n_mel = int(self.noise.shape[1] * top / self.model_sr) // ehop + 4
            self.gen_rand_ini = torch.zeros(1, 1, SINEGEN_DIM, device=dev)
            self.gen_noise = torch.zeros(1, n_mel * ehop, SINEGEN_DIM, device=dev)
            self.enhancer.prepare(self.model_sr, [self.key] if self.key != "auto" else range(self.max_key() + 1))
        self.ratio_host = torch.zeros(1, dtype=torch.float32).pin_memory()
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
        self._draw_sinegen(self.gen_rand_ini, self.gen_noise)

    # ---- the two halves of the block ----------------------------------------------------------------------------------
    def _stage_a(self):
        """ring buffer -> masked synthesizer output [1, T] and max(f0[start_frame:]) / 760"""
        f0, volume, mask, units = self._front()
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
        self._tail(out, self.out_sr)

    # ---- one callback -------------------------------------------------------------------------------------------------
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
        return self._output()


class RealtimeReflowVC(_Session):
    """gui_reflow.py's block on the reflow model (see the module's docstring).  One deviation from the reference:
    gui_reflow.py:137 hands spk_mix_dict to the model whether or not use_spk_mix is set; the session mixes speakers only
    with use_spk_mix, as gui.py and RealtimeVC do."""

    def __init__(self, model_path, samplerate=44100, block_time=0.5, crossfade_time=0.04, extra_time=2.0, f0_min=50,
                 f0_max=1100, threhold=-45, spk_id=1, pitch_adjust=0.0, formant_shift_key=0.0, use_spk_mix=False,
                 spk_mix_dict=None, use_phase_vocoder=False, t_start=0.7, infer_step=30, sampling_method="euler",
                 graph=True, pitch_extractor_type="rmvpe", rmvpe_ckpt="pretrain/rmvpe/model.pt", device=None):
        if pitch_extractor_type != "rmvpe":
            raise ValueError("RealtimeReflowVC extracts f0 with 'rmvpe' only: %r has no kernels"
                             % (pitch_extractor_type,))
        if int(infer_step) != infer_step or infer_step < 1:
            raise ValueError("infer_step must be an integer >= 1, got %r" % (infer_step,))
        if sampling_method not in ("euler", "rk4"):
            raise ValueError("sampling_method must be 'euler' or 'rk4', got %r" % (sampling_method,))
        self._init_block(samplerate, block_time, crossfade_time, extra_time, device, "RealtimeReflowVC")
        self.f0_max = float(f0_max)
        self.formant_shift_key, self.t_start = float(formant_shift_key), float(t_start)
        self.infer_step, self.method = int(infer_step), sampling_method
        self.use_pv, self.graph = bool(use_phase_vocoder), bool(graph)

        self.model, self.vocoder, self.args = load_model_vocoder(model_path, device=self.device)
        data = self.args.data
        self.frames = reflow_frames(self.sr, block_time, crossfade_time, extra_time, int(data.sampling_rate),
                                    int(data.block_size), self.vocoder.vocoder_hop_size, self.vocoder.h.win_size)
        self._init_front(data, f0_min, threhold, pitch_adjust, spk_id, use_spk_mix, spk_mix_dict, rmvpe_ckpt,
                         "RealtimeReflowVC")
        self.mask_offset = self.frames["mask_offset"]

        dev, T = self.device, self.frames["mel_frames"]
        self.aug_shift = torch.tensor([[self.formant_shift_key]], dtype=torch.float32, device=dev)
        self.noise = torch.zeros(1, self.n_frames * self.block_size, device=dev)      # CombSubSuperFast: randn
        self.reflow_noise = torch.zeros(1, 1, self.vocoder.dimension, T, device=dev)
        self.gen_rand_ini = torch.zeros(1, 1, SINEGEN_DIM, device=dev)
        self.gen_noise = torch.zeros(1, T * self.vocoder.vocoder_hop_size, SINEGEN_DIM, device=dev)
        self.graph_block = None

    def _draw_noise(self):
        """the block's draws: the DDSP noise, the sampler's initial noise, SineGen's rand_ini and noise"""
        self.noise.normal_()
        self.reflow_noise.normal_()
        self._draw_sinegen(self.gen_rand_ini, self.gen_noise)

    def _stage(self):
        f0, volume, mask, units = self._front()
        self._draw_noise()
        with torch.no_grad():
            out = self.model(units, f0, volume[..., None], spk_id=self.spk_id, spk_mix_dict=self.spk_mix_dict,
                             aug_shift=self.aug_shift, vocoder=self.vocoder, infer=True, return_wav=True,
                             infer_step=self.infer_step, method=self.method, t_start=self.t_start,
                             silence_front=self.silence_front, use_tqdm=False, ddsp_noise=self.noise,
                             reflow_noise=self.reflow_noise, rand_ini=self.gen_rand_ini, sine_noise=self.gen_noise)
        out = frontend.mask_apply_(out.reshape(1, -1).contiguous(), mask, self.block_size, self.mask_offset)
        self._tail(out, self.model_sr)

    def run(self):
        """enqueue the block's graph (or its eager code) on the session's stream"""
        if not self.graph:
            with torch.cuda.stream(self.stream):
                self._stage()
            return
        if self.graph_block is None:
            self.graph_block, _ = self._capture(self._stage, [self.ring, self.sola_buffer])
        with torch.cuda.stream(self.stream):
            self.graph_block.replay()

    def process(self, indata):
        """audio_callback's math: indata [frames, channels] -> outdata [frames, 2] (float32)"""
        self.upload(indata)
        self.run()
        return self._output()
