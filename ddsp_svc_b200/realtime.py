"""The real-time conversion blocks of gui.py, gui_reflow.py and gui_diff.py on the device, replayed as CUDA graphs.

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

``RealtimeDiffVC(model_path, diff_model_path, ..., k_step, diff_acc, diff_method, diff_silence, ...)`` is gui_diff.py's
block (audio_callback, gui_diff.py:437-503, with SvcDDSP.update_model / infer, :48-154) on the diffusion cascade
(diffusion_vocoder): ring buffer -> RMVPE -> rt_f0_regrid -> volume -> mask -> units -> the DDSP model -> DiffGtMel.infer
(the mel of the DDSP output, the shallow-diffusion sampler from k_step, the crop at its start_frame or the diff_silence
input crop, NSF-HiFiGAN) -> mask multiply -> resampling -> rt_sola -> rt_crossfade -> pinned copy, ONE graph.  Its draws
(the DDSP noise, the sampler's start, DDPM's per-step noise, SineGen's rand_ini and noise) are static buffers filled by
torch's CUDA generator, and GaussianDiffusion keeps its step rows and coefficients after the warm-up.

The sessions share ``_Session``: the ring buffer, the upload and the owned stream, capture with a warm-up and a state
restore, the f0 / volume / mask / units front half, the resampling -> SOLA -> crossfade -> pinned-copy tail and
SineGen's draws.  ``reflow_frames`` and ``diff_frames`` are the reflow and diffusion blocks' frame bookkeeping as pure
functions.
"""
import gc

import numpy as np
import torch

from . import frontend, ops
from .diffusion_vocoder import DiffGtMel, Unit2WavFast, read_config
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


def units_encoder(data, device):
    """the checkpoint config's data section -> its Units_Encoder, built as main.py and the GUIs build it (the
    cnhubertsoft_gate from the config, 10 without one)"""
    return Units_Encoder(data.encoder, data.encoder_ckpt, data.encoder_sample_rate, data.encoder_hop_size, device=device,
                         cnhubertsoft_gate=getattr(data, "cnhubertsoft_gate", None) or 10)


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


def _mel_frames(n, vocoder_hop, win_size):
    """the frames nvSTFT.get_mel makes of n samples (its reflect-or-constant padding, center=False)"""
    pad_left = (win_size - vocoder_hop) // 2
    pad_right = max((win_size - vocoder_hop + 1) // 2, win_size - n - pad_left)
    return (n + pad_left + pad_right - win_size) // vocoder_hop + 1


def diff_frames(samplerate, block_time, crossfade_time, extra_time, model_sr, block_size, vocoder_sr, vocoder_hop,
                win_size=2048, diff_silence=False):
    """The frame bookkeeping of one gui_diff.py block -> dict:

    - gui_frames' lengths and silence_front; ``hop`` and ``n_frames`` (F0_Extractor's and the volume's frames);
    - ``start_frame`` / ``trim``: F0_Extractor's leading frames and the samples RMVPE skips;
    - ``diff_start``: DiffGtMel.infer's start_frame, int(silence_front * vocoder rate / vocoder hop);
    - ``cond_frames``: the frames the diffusion model sees (n_frames, or n_frames - diff_start with diff_silence), which
      are also its mel frames; ``voc_frames``: the frames vocoded (from diff_start on);
    - ``out_len``: the output's samples at the model rate after the left pad (n_frames block_size), ``out_dev`` its
      length at the device rate and ``tail``: the (start, stop) of the samples SOLA reads.
    Raises ValueError where the reference's block cannot run: a non-integer hop, a vocoder rate or hop other than the
    model's (``output *= mask`` would not broadcast), or a mel whose frame count differs from the condition's."""
    f = gui_frames(samplerate, block_time, crossfade_time, extra_time)
    sr = f["sr"]
    hop = model_hop(sr, model_sr, block_size, "RealtimeDiffVC")
    if vocoder_sr != model_sr or vocoder_hop != block_size:
        raise ValueError("the vocoder runs at %d Hz with hop %d, the model at %d Hz with block_size %d: gui_diff.py's "
                         "output *= mask needs both equal" % (vocoder_sr, vocoder_hop, model_sr, block_size))
    n_frames = f["n_in"] // hop + 1
    start_frame = int(f["silence_front"] * sr / hop)
    diff_start = int(f["silence_front"] * vocoder_sr / vocoder_hop)
    cond_frames = n_frames - diff_start if diff_silence else n_frames
    mel_frames = _mel_frames(cond_frames * block_size, vocoder_hop, win_size)
    if mel_frames != cond_frames:
        raise ValueError("the mel of %d DDSP frames has %d frames: the diffusion model's condition has %d"
                         % (cond_frames, mel_frames, cond_frames))
    out_len = n_frames * vocoder_hop
    out_dev = out_len if model_sr == sr else resampled_length(out_len, model_sr, sr)
    tail = (out_dev - f["block"] - f["cf"] - f["search"] - f["delay"], out_dev - f["delay"])
    f.update(hop=hop, n_frames=n_frames, start_frame=start_frame, trim=int(np.round(start_frame * hop / sr * sr)),
             diff_start=diff_start, cond_frames=cond_frames, mel_frames=mel_frames, voc_frames=n_frames - diff_start,
             out_len=out_len, out_dev=out_dev, tail=tail)
    return f


class _Session:
    """What the real-time sessions share (see the module's docstring)"""

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
        self.units_encoder = units_encoder(data, dev)
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
        warm-up's writes to the session state tensors are undone, so the first replay starts where it should.

        Python's cycle collector does not run during the capture: it could free an unreachable CUDAGraph (another
        session's, dropped while in a reference cycle), and destroying a graph while a stream captures is an operation
        CUDA forbids, which corrupts this capture.  Garbage is collected just before instead (torch.cuda.graph no
        longer does that by default)."""
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            saved = [t.clone() for t in state]
            fn()
            for t, v in zip(state, saved):
                t.copy_(v)
        self.stream.synchronize()
        collecting = gc.isenabled()
        gc.collect()
        gc.disable()
        try:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=self.stream):
                static = fn()
        finally:
            if collecting:
                gc.enable()
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


DIFF_METHODS = ("ddim", "pndm", "dpm-solver", "unipc")


class RealtimeDiffVC(_Session):
    """gui_diff.py's block on the diffusion models (see the module's docstring).  ``model_path`` is the DDSP checkpoint
    (None or '' for none), ``diff_model_path`` the diffusion model's.  A 'Diffusion' model (Unit2Mel) starts its sampler
    from the DDSP output's mel at k_step; without a DDSP checkpoint it samples from noise from GaussianDiffusion.k_step
    (1000), as the reference does.  diff_acc 1 samples with DDPM.

    Deviations from the reference: for 'DiffusionNew' / 'DiffusionFast', Unit2Wav computes its own DDSP mel and ignores
    the external DDSP output, so the session checks the DDSP checkpoint's config against the diffusion model's but does
    not run it; and, as in the other sessions, a speaker mix applies only with use_spk_mix."""

    def __init__(self, model_path, diff_model_path, samplerate=44100, block_time=0.5, crossfade_time=0.04,
                 extra_time=2.0, f0_min=50, f0_max=1100, threhold=-45, spk_id=1, pitch_adjust=0.0, use_spk_mix=False,
                 spk_mix_dict=None, use_phase_vocoder=False, k_step=100, diff_acc=10, diff_method="ddim",
                 diff_silence=False, graph=True, pitch_extractor_type="rmvpe", rmvpe_ckpt="pretrain/rmvpe/model.pt",
                 device=None):
        if pitch_extractor_type != "rmvpe":
            raise ValueError("RealtimeDiffVC extracts f0 with 'rmvpe' only: %r has no kernels" % (pitch_extractor_type,))
        if diff_method not in DIFF_METHODS:
            raise ValueError("diff_method must be one of %s, got %r" % (", ".join(DIFF_METHODS), diff_method))
        if int(k_step) != k_step or k_step < 0:
            raise ValueError("k_step must be an integer >= 0, got %r" % (k_step,))
        if int(diff_acc) != diff_acc or (k_step > 0 and not 1 <= diff_acc <= k_step // 2):
            raise ValueError("diff_acc must be an integer in [1, k_step // 2] = [1, %d] (1: DDPM), got %r"
                             % (int(k_step) // 2, diff_acc))
        self._init_block(samplerate, block_time, crossfade_time, extra_time, device, "RealtimeDiffVC")
        self.f0_max = float(f0_max)
        self.k_step, self.diff_acc, self.diff_method = int(k_step), int(diff_acc), diff_method
        self.diff_silence, self.use_pv, self.graph = bool(diff_silence), bool(use_phase_vocoder), bool(graph)

        # SvcDDSP.update_model: the DDSP checkpoint's config is checked against the diffusion model's (check_args)
        args = read_config(diff_model_path)
        kind = args.model.type
        k_step_max = int(args.model.k_step_max) if kind == "DiffusionNew" else 1000
        if self.k_step > k_step_max:
            raise ValueError("k_step %d exceeds the model's k_step_max %d" % (self.k_step, k_step_max))
        if kind == "Diffusion" and self.k_step == 0:
            raise ValueError("a 'Diffusion' model needs k_step >= 1: its shallow start noises to step k_step - 1")
        self.diff = DiffGtMel(device=self.device)
        ddsp_args = read_config(model_path) if model_path else None
        if ddsp_args is not None:
            self.diff.check_args(ddsp_args, args)
        self.diff.flush_model(diff_model_path, ddsp_config=ddsp_args)
        self.model, self.vocoder, self.args = self.diff.model, self.diff.vocoder, self.diff.args
        self.ddsp_model = None
        if kind == "Diffusion" and model_path:
            self.ddsp_model, self.ddsp_args = load_model(model_path, device=self.device)
        data = self.args.data
        self.frames = diff_frames(self.sr, block_time, crossfade_time, extra_time, int(data.sampling_rate),
                                  int(data.block_size), self.vocoder.vocoder_sample_rate, self.vocoder.vocoder_hop_size,
                                  self.vocoder.h.win_size, self.diff_silence)
        self._init_front(data, f0_min, threhold, pitch_adjust, spk_id, use_spk_mix, spk_mix_dict, rmvpe_ckpt,
                         "RealtimeDiffVC")

        dev, fr, M = self.device, self.frames, self.vocoder.dimension
        T = fr["cond_frames"]
        self.ext_noise = None                 # the external DDSP model's noise: randn for CombSubSuperFast, else uniform
        if self.ddsp_model is not None:
            self.ext_noise = torch.zeros(1, self.n_frames * self.block_size, device=dev)
            self.ext_normal = self.ddsp_args.model.type == "CombSubSuperFast"
        self.ddsp_noise = None                # Unit2Wav's CombSubFast (uniform) / Unit2WavFast's CombSubSuperFast (randn)
        if kind != "Diffusion":
            self.ddsp_noise = torch.zeros(1, T * self.block_size, device=dev)
        # the sampler's start: with a gt_spec, randn_like of the transposed [B, 1, M, T] view; without, torch.randn
        has_gt = kind != "Diffusion" or self.ddsp_model is not None
        runs = kind == "Diffusion" or self.k_step > 0
        self.diff_noise = self.step_noise = None
        if runs:
            self.diff_noise = (torch.empty_strided((1, 1, M, T), (T * M, T * M, 1, M), device=dev) if has_gt else
                               torch.empty(1, 1, M, T, device=dev)).zero_()
            if self.diff_acc == 1:
                n_steps = self.k_step if has_gt else self.model.decoder.k_step
                self.step_noise = torch.zeros(n_steps, 1, 1, M, T, device=dev)
        self.gen_rand_ini = torch.zeros(1, 1, SINEGEN_DIM, device=dev)
        self.gen_noise = torch.zeros(1, fr["voc_frames"] * self.vocoder.vocoder_hop_size, SINEGEN_DIM, device=dev)
        self.graph_block = None

    def _draw_noise(self):
        """the block's draws: the DDSP noise, the sampler's start, DDPM's per-step noise, SineGen's rand_ini and noise"""
        if self.ext_noise is not None:
            if self.ext_normal:
                self.ext_noise.normal_()
            else:
                self.ext_noise.uniform_(-1, 1)
        if self.ddsp_noise is not None:
            if isinstance(self.model, Unit2WavFast):
                self.ddsp_noise.normal_()
            else:
                self.ddsp_noise.uniform_(-1, 1)
        if self.diff_noise is not None:
            self.diff_noise.normal_()
        if self.step_noise is not None:
            self.step_noise.normal_()
        self._draw_sinegen(self.gen_rand_ini, self.gen_noise)

    def draws(self):
        """the draws DiffGtMel.infer takes, from the static buffers"""
        d = dict(noise=self.diff_noise, step_noise=self.step_noise, rand_ini=self.gen_rand_ini, sine_noise=self.gen_noise)
        if self.ddsp_noise is not None:
            d["ddsp_noise"] = self.ddsp_noise
        return d

    def _stage(self):
        f0, volume, mask, units = self._front()
        self._draw_noise()
        with torch.no_grad():
            out = None
            if self.ddsp_model is not None:
                out, _, _ = self.ddsp_model(units, f0, volume[..., None], spk_id=self.spk_id,
                                            spk_mix_dict=self.spk_mix_dict, noise=self.ext_noise)
            out = self.diff.infer(out, f0, units, volume[..., None], acc=self.diff_acc, spk_id=self.spk_id,
                                  k_step=self.k_step, method=self.diff_method, silence_front=self.silence_front,
                                  use_silence=self.diff_silence, spk_mix_dict=self.spk_mix_dict, **self.draws())
        out = frontend.mask_apply_(out.reshape(1, -1).contiguous(), mask, self.block_size)
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
