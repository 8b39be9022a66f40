"""The whole-file conversion of main.py and main_reflow.py on the device: the Slicer's cut, every segment's model call
and the cross-faded assembly, queued on one stream without a host round trip per segment.

``OfflineVC(model_path, device=None, enhance=True, rmvpe_ckpt=...)`` is main.py (its lines after the argument parsing,
with the DDSP model of ``load_model`` and the ``Enhancer``); ``OfflineReflowVC(model_path, device=None, rmvpe_ckpt=...)``
is main_reflow.py (``load_model_vocoder``'s Unit2Wav and its vocoder).  Both take mono CUDA fp32 audio [N] and return
CUDA fp32 audio [N_out] with its sample rate; file I/O and the f0 cache stay with the caller.

- ``split(audio, sample_rate)`` -> [(start_frame, end_frame)]: main.py's ``split()`` (db_thresh -40, min_len 5000 ms).
  The Slicer's frame RMS is ``frontend.slicer_rms`` on the device, copied back once; its silence state machine and
  main.py's frame arithmetic are the host functions ``silence_tags``, ``slicer_chunks`` and ``split_frames``.
- ``convert(audio, sample_rate, ..., segments=None)``: f0 for the whole file (RMVPE, then ``ops.rt_f0_regrid``:
  F0_Extractor's 'rmvpe' post-processing with uv_interp and the key's pitch factor), volume and mask for the whole
  file, then per segment, in main.py's order: units of a view of the segment, f0 / volume sliced to its unit frames,
  the model, the mask at the segment's frame offset and the enhancer (main.py) or the vocoder (main_reflow.py).
  ``frontend.segment_place_`` writes each output into the zero-filled result with main.py's fade; ``assembly_plan``
  is main.py's integer bookkeeping (``silent_length`` / ``current_length``), which needs only the output lengths.
  With ``segments`` given and a numeric ``enhancer_adaptive_key``, the call queues all its work without a host
  synchronisation; ``'auto'`` reads one scalar per segment, as the reference's Enhancer does.
- ``render(...)`` is ``convert`` without the assembly: the segments' outputs, for callers that place them themselves.

Only 'rmvpe' f0 and integer hops (block_size * sample_rate / sampling_rate) are supported: the volume kernel needs an
integer hop, as in the real-time sessions.
"""
import numpy as np
import torch

from . import frontend, ops
from .dropin import load_model
from .enhancer import Enhancer
from .realtime import model_hop, units_encoder
from .reflow_vocoder import load_model_vocoder
from .rmvpe import RMVPE

# main.py's split(): Slicer(sr, threshold=db_thresh, min_length=min_len) with its other defaults
DB_THRESH, MIN_LEN_MS, MIN_INTERVAL_MS, HOP_MS, MAX_SIL_KEPT_MS = -40.0, 5000, 300, 20, 5000


class SlicerParams:
    """the reference Slicer's constructor arithmetic at sample rate sr: hop and win in samples, the threshold as an
    amplitude, min_length / min_interval / max_sil_kept in frames"""

    def __init__(self, sr, threshold=DB_THRESH, min_length=MIN_LEN_MS, min_interval=MIN_INTERVAL_MS, hop_size=HOP_MS,
                 max_sil_kept=MAX_SIL_KEPT_MS):
        interval = sr * min_interval / 1000
        self.threshold = 10 ** (threshold / 20.)
        self.hop = round(sr * hop_size / 1000)
        self.win = min(round(interval), 4 * self.hop)
        self.min_length = round(sr * min_length / 1000 / self.hop)
        self.min_interval = round(interval / self.hop)
        self.max_sil_kept = round(sr * max_sil_kept / 1000 / self.hop)


def silence_tags(rms, p):
    """The Slicer's silence state machine over the frame RMS -> [(first, last)] frame pairs of the silences it cuts.

    A silent run is a stretch of frames with rms below the threshold (compared in fp32, as numpy compares the fp32
    rms with the Python float).  It is cut when it is leading silence longer than max_sil_kept, or when it lasts at
    least min_interval frames and the clip before it at least min_length.  Runs of up to max_sil_kept frames collapse
    to their quietest frame; up to twice that keep max_sil_kept frames on each side around it; longer ones keep
    max_sil_kept frames at each end.  "Quietest" is argmin's first minimum.  A trailing run of at least min_interval
    frames is cut from the quietest of its first max_sil_kept + 1 frames to total_frames + 1."""
    rms = np.asarray(rms, dtype=np.float32)
    quiet = rms < np.float32(p.threshold)
    k = p.max_sil_kept

    def quietest(a, b):
        return a + int(np.argmin(rms[a:b]))

    tags, run, clip = [], None, 0
    for i in range(rms.shape[0]):
        if quiet[i]:
            run = i if run is None else run
            continue
        if run is None:
            continue
        leading = run == 0 and i > k
        middle = i - run >= p.min_interval and i - clip >= p.min_length
        if leading or middle:
            if i - run <= k:
                pos = quietest(run, i + 1)
                tags.append((0 if run == 0 else pos, pos))
                clip = pos
            elif i - run <= 2 * k:
                pos = quietest(i - k, run + k + 1)
                left, right = quietest(run, run + k + 1), quietest(i - k, i + 1)
                tags.append((0, right) if run == 0 else (min(left, pos), max(right, pos)))
                clip = right if run == 0 else max(right, pos)
            else:
                left, right = quietest(run, run + k + 1), quietest(i - k, i + 1)
                tags.append((0 if run == 0 else left, right))
                clip = right
        run = None
    n = rms.shape[0]
    if run is not None and n - run >= p.min_interval:
        tags.append((quietest(run, min(n, run + k) + 1), n + 1))
    return tags


def slicer_chunks(tags, n_samples, hop):
    """the Slicer's chunks [(begin, end, silent)] in samples from its silence tags: the voiced stretches between the
    silences and the silences themselves, ends clipped to the signal (one voiced chunk when nothing is cut)"""
    if not tags:
        return [(0, n_samples, False)]
    chunks = [(0, min(n_samples, tags[0][0] * hop), False)] if tags[0][0] else []
    for i, (first, last) in enumerate(tags):
        if i:
            chunks.append((tags[i - 1][1] * hop, min(n_samples, first * hop), False))
        chunks.append((first * hop, min(n_samples, last * hop), True))
    if tags[-1][1] * hop < n_samples:
        chunks.append((tags[-1][1] * hop, n_samples, False))
    return chunks


def split_frames(chunks, hop_size):
    """main.py's split() on the Slicer's chunks -> [(start_frame, end_frame)] at the model's hop: every chunk, silent
    ones included, that spans at least one whole frame"""
    out = []
    for begin, end, _ in chunks:
        if begin != end:
            start, stop = int(begin // hop_size), int(end // hop_size)
            if stop > start:
                out.append((start, stop))
    return out


def assembly_plan(start_frames, lengths, block_size, out_sr, model_sr):
    """main.py's assembly bookkeeping for segment outputs of these lengths -> ([(idx, fade_len)], total length): a
    segment goes at round(start_frame block_size out_sr / model_sr) and cross-fades over what the previous ones wrote
    past that point.  Raises ValueError where main.py's cross_fade would fail: a fade longer than the segment."""
    plan, current = [], 0
    for start, n in zip(start_frames, lengths):
        silent = round(start * block_size * out_sr / model_sr) - current
        fade = max(0, -silent)
        if fade > n:
            raise ValueError("the segment at frame %d holds %d samples but would cross-fade over the last %d samples "
                             "written: main.py's cross_fade cannot broadcast that" % (start, n, fade))
        plan.append((current + silent, fade))
        current += silent + n
    return plan, current


def _need_audio(audio):
    if not (isinstance(audio, torch.Tensor) and audio.is_cuda and audio.dtype == torch.float32 and audio.dim() == 1):
        raise ValueError("audio must be a mono [N] CUDA float32 tensor")


class _Offline:
    """What OfflineVC and OfflineReflowVC share: the front (RMVPE, units encoder), split, the whole-file f0 / volume
    / mask, the per-segment inputs and the assembly"""

    def _init_device(self, device, pitch_extractor, who):
        if pitch_extractor != "rmvpe":
            raise ValueError("%s extracts f0 with 'rmvpe' only: %r has no kernels" % (who, pitch_extractor))
        self.device = torch.device("cuda" if device is None else device)
        if self.device.type != "cuda":
            raise ValueError("%s runs on the CUDA kernels: device must be a CUDA device" % who)
        self.who = who

    def _init_front(self, data, rmvpe_ckpt):
        self.model_sr, self.block_size = int(data.sampling_rate), int(data.block_size)
        self.units_encoder = units_encoder(data, self.device)
        self.rmvpe = RMVPE(rmvpe_ckpt, hop_length=160)

    def hop(self, sample_rate):
        """block_size * sample_rate / sampling_rate, which must be an integer"""
        return model_hop(int(sample_rate), self.model_sr, self.block_size, self.who)

    def split(self, audio, sample_rate):
        """main.py's split(audio, sample_rate, hop_size) -> [(start_frame, end_frame)]; reads the frame RMS back once"""
        _need_audio(audio)
        hop = self.hop(sample_rate)
        p = SlicerParams(int(sample_rate))
        n = audio.shape[0]
        if n <= p.min_length:                   # the Slicer compares the sample count with min_length in frames
            tags = []
        else:
            with torch.cuda.device(audio.device):
                rms = frontend.slicer_rms(audio, p.win, p.hop).cpu().numpy()
            tags = silence_tags(rms, p)
        return split_frames(slicer_chunks(tags, n, p.hop), hop)

    def _front(self, audio, sample_rate, key, f0_min, threhold):
        """the whole file's f0 [1, nF, 1] (key applied), volume [1, nF] and mask [1, nF]"""
        hop = self.hop(sample_rate)
        n_frames = audio.shape[0] // hop + 1
        x = audio[None]
        f0_10ms = self.rmvpe.infer_batch(x, sample_rate)[0]
        f0 = ops.rt_f0_regrid(f0_10ms.contiguous(), 0.01, n_frames, hop / sample_rate, rmvpe=True, pad=0,
                              f0_min=float(f0_min), post_scale=2 ** (float(key) / 12))
        volume = frontend.volume_extract(x, hop)
        mask = frontend.volume_mask(volume, float(threhold))
        return f0[None, :, None], volume, mask

    def _segments(self, audio, sample_rate, key, f0_min, threhold, segments):
        """yields (start_frame, units, f0, volume, mask) of each segment, main.py's slices"""
        hop = self.hop(sample_rate)
        if segments is None:
            segments = self.split(audio, sample_rate)
        f0, volume, mask = self._front(audio, sample_rate, key, f0_min, threhold)
        for start, stop in segments:
            start, stop = int(start), int(stop)
            if not 0 <= start < stop <= audio.shape[0] // hop:
                raise ValueError("segment (%d, %d) is not a frame range of the %d-frame audio"
                                 % (start, stop, audio.shape[0] // hop))
            units = self.units_encoder.encode(audio[None, start * hop:stop * hop], sample_rate, hop)
            n = units.size(1)
            yield start, units, f0[:, start:start + n, :], volume[:, start:start + n, None], mask

    def _mask(self, out, mask, start):
        return frontend.mask_apply_(out.reshape(1, -1).contiguous(), mask, self.block_size, start)

    def _spk_id(self, spk_id):
        return torch.full((1, 1), int(spk_id), dtype=torch.long, device=self.device)

    def assemble(self, rendered, out_sr):
        """[(start_frame, output [T])] -> the whole-file output [N_out]: main.py's assembly on the device"""
        plan, total = assembly_plan([s for s, _ in rendered], [o.numel() for _, o in rendered], self.block_size,
                                    out_sr, self.model_sr)
        result = torch.zeros(total, dtype=torch.float32, device=self.device)
        for (_, out), (idx, fade) in zip(rendered, plan):
            frontend.segment_place_(result, out.reshape(-1), idx, fade)
        return result

    def convert(self, audio, sample_rate, *args, **kwargs):
        rendered, out_sr = self.render(audio, sample_rate, *args, **kwargs)
        with torch.cuda.device(self.device):
            return self.assemble(rendered, out_sr), out_sr


class OfflineVC(_Offline):
    """main.py's conversion on the DDSP model of ``load_model`` and, with ``enhance``, the NSF-HiFiGAN ``Enhancer``"""

    def __init__(self, model_path, device=None, enhance=True, rmvpe_ckpt="pretrain/rmvpe/model.pt",
                 pitch_extractor="rmvpe"):
        self._init_device(device, pitch_extractor, "OfflineVC")
        self.model, self.args = load_model(model_path, device=self.device)
        self._init_front(self.args.data, rmvpe_ckpt)
        self.enhancer = Enhancer(self.args.enhancer.type, self.args.enhancer.ckpt, self.device) if enhance else None

    def render(self, audio, sample_rate, key=0, spk_id=1, spk_mix_dict=None, f0_min=50, f0_max=1100, threhold=-60,
               enhancer_adaptive_key=0, segments=None):
        """convert() without the assembly -> ([(start_frame, output [T])], output sample rate).  f0_max is accepted
        for main.py's signature: RMVPE's f0 is not bounded above"""
        _need_audio(audio)
        sample_rate = int(sample_rate)
        out_sr = self.enhancer.enhancer_sample_rate if self.enhancer is not None else self.model_sr
        rendered = []
        with torch.cuda.device(self.device), torch.no_grad():
            spk = self._spk_id(spk_id)
            for start, units, f0, volume, mask in self._segments(audio, sample_rate, key, f0_min, threhold, segments):
                out, _, _ = self.model(units, f0, volume, spk_id=spk, spk_mix_dict=spk_mix_dict)
                out = self._mask(out, mask, start)
                if self.enhancer is not None:
                    out, _ = self.enhancer.enhance(out, self.model_sr, f0, self.block_size,
                                                   adaptive_key=enhancer_adaptive_key)
                rendered.append((start, out.reshape(-1)))
        return rendered, out_sr

    def convert(self, audio, sample_rate, key=0, spk_id=1, spk_mix_dict=None, f0_min=50, f0_max=1100, threhold=-60,
                enhancer_adaptive_key=0, segments=None):
        """main.py's whole-file conversion -> (output [N_out] CUDA fp32, its sample rate)"""
        return super().convert(audio, sample_rate, key=key, spk_id=spk_id, spk_mix_dict=spk_mix_dict, f0_min=f0_min,
                               f0_max=f0_max, threhold=threhold, enhancer_adaptive_key=enhancer_adaptive_key,
                               segments=segments)


def reflow_settings(args, infer_step="auto", method="auto", t_start="auto"):
    """main_reflow.py's sampler settings -> (infer_step, method, t_start): 'auto' from the config's infer section and
    model.t_start (0 without one); a given t_start is raised to model.t_start.  A negative infer_step raises"""
    def infer(key):
        section = args.infer
        if section is None or section.get(key) is None:
            raise ValueError("%s='auto' needs infer.%s in the model's config" % (key, key))
        return section.get(key)

    method = infer("method") if method == "auto" else method
    infer_step = int(infer("infer_step")) if infer_step == "auto" else int(infer_step)
    floor = args.model.t_start
    if t_start == "auto":
        t_start = float(floor) if floor is not None else 0.0
    else:
        t_start = float(t_start)
        if floor is not None and t_start < floor:
            t_start = float(floor)
    if infer_step < 0:
        raise ValueError("infer_step cannot be negative, got %d" % infer_step)
    if method not in ("euler", "rk4"):
        raise ValueError("method must be 'euler' or 'rk4', got %r" % (method,))
    return infer_step, method, t_start


class OfflineReflowVC(_Offline):
    """main_reflow.py's conversion on ``load_model_vocoder``'s Unit2Wav and its vocoder"""

    def __init__(self, model_path, device=None, rmvpe_ckpt="pretrain/rmvpe/model.pt", pitch_extractor="rmvpe"):
        self._init_device(device, pitch_extractor, "OfflineReflowVC")
        self.model, self.vocoder, self.args = load_model_vocoder(model_path, device=self.device)
        self._init_front(self.args.data, rmvpe_ckpt)

    def render(self, audio, sample_rate, key=0, spk_id=1, spk_mix_dict=None, f0_min=50, f0_max=1100, threhold=-60,
               formant_shift_key=0, infer_step="auto", method="auto", t_start="auto", segments=None):
        """convert() without the assembly -> ([(start_frame, output [T])], the model's sample rate)"""
        _need_audio(audio)
        sample_rate = int(sample_rate)
        infer_step, method, t_start = reflow_settings(self.args, infer_step, method, t_start)
        rendered = []
        with torch.cuda.device(self.device), torch.no_grad():
            spk = self._spk_id(spk_id)
            aug_shift = torch.full((1, 1), float(formant_shift_key), dtype=torch.float32, device=self.device)
            for start, units, f0, volume, mask in self._segments(audio, sample_rate, key, f0_min, threhold, segments):
                out = self.model(units, f0, volume, spk_id=spk, spk_mix_dict=spk_mix_dict, aug_shift=aug_shift,
                                 vocoder=self.vocoder, infer=True, return_wav=True, infer_step=infer_step,
                                 method=method, t_start=t_start, use_tqdm=False)
                rendered.append((start, self._mask(out, mask, start).reshape(-1)))
        return rendered, self.model_sr

    def convert(self, audio, sample_rate, key=0, spk_id=1, spk_mix_dict=None, f0_min=50, f0_max=1100, threhold=-60,
                formant_shift_key=0, infer_step="auto", method="auto", t_start="auto", segments=None):
        """main_reflow.py's whole-file conversion -> (output [N_out] CUDA fp32, the model's sample rate)"""
        return super().convert(audio, sample_rate, key=key, spk_id=spk_id, spk_mix_dict=spk_mix_dict, f0_min=f0_min,
                               f0_max=f0_max, threhold=threhold, formant_shift_key=formant_shift_key,
                               infer_step=infer_step, method=method, t_start=t_start, segments=segments)
