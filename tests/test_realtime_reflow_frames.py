"""Without a GPU: the package's Unit2Wav has the reference's parameter tree (tests/golden/unit2wav_state_dicts.json) and
loads it strictly, RealtimeReflowVC's argument checks, and reflow_frames (ddsp_svc_b200/realtime.py), the gui_reflow.py
block's frame bookkeeping, pinned against gui_reflow.py's own formulas restated here: GUI.set_values, SvcDDSP.infer's
silence_front, F0_Extractor's frames and trim, Unit2Wav's start_frame, nvSTFT's frames (torch.stft with its padding),
the ``mask[:, -output.shape[-1]:]`` slice and the SOLA window of audio_callback after torchaudio's resampling."""
import json
import os

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200.realtime import RealtimeReflowVC, reflow_frames

HERE = os.path.dirname(os.path.abspath(__file__))
MODEL_SR, BLOCK_SIZE, VOC_HOP, WIN = 44100, 512, 512, 2048


@pytest.mark.parametrize("model,n_layers,n_chans", [("w128", 2, 128), ("w512", 6, 512)])
def test_unit2wav_has_the_reference_tree(model, n_layers, n_chans):
    with open(os.path.join(HERE, "golden", "unit2wav_state_dicts.json")) as f:
        ref = json.load(f)[model]
    net = pkg.Unit2Wav(MODEL_SR, BLOCK_SIZE, 2048, 256, 2, True, 128, n_layers, n_chans)
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == ref
    sd = {k: torch.full(shape, 0.5) for k, shape in ref}
    net.load_state_dict(sd, strict=True)
    assert net.reflow_model.velocity_fn.output_projection.weight.detach().eq(0.5).all()


def test_unit2wav_refuses_training():
    net = pkg.Unit2Wav(MODEL_SR, BLOCK_SIZE, 2048, 256, 1, False, 128, 1, 64)
    with pytest.raises(NotImplementedError, match="patch_reference"):
        net(None, None, None, infer=False)


@pytest.mark.parametrize("kw,match", [(dict(pitch_extractor_type="crepe"), "rmvpe"), (dict(infer_step=0), "infer_step"),
                                      (dict(infer_step=2.5), "infer_step"), (dict(sampling_method="heun"), "heun")])
def test_session_arguments_checked_before_loading(kw, match):
    with pytest.raises(ValueError, match=match):
        RealtimeReflowVC("no/such/model.pt", **kw)


def gui_reflow(samplerate, block_time, crossfade_time, extra_time):
    """gui_reflow.py's own arithmetic for one block"""
    block_frame = int(block_time * samplerate)
    crossfade_frame = int(crossfade_time * samplerate)
    sola_search_frame = int(0.01 * samplerate)
    last_delay_frame = int(0.02 * samplerate)
    extra_frame = int(extra_time * samplerate)
    input_frame = max(block_frame + crossfade_frame + sola_search_frame + 2 * last_delay_frame,
                      block_frame + extra_frame)
    f_safe_prefix_pad_length = extra_time - crossfade_time - 0.01 - 0.02
    silence_front = f_safe_prefix_pad_length - 0.03 if f_safe_prefix_pad_length > 0.03 else 0
    hop_size = BLOCK_SIZE * samplerate / MODEL_SR
    audio = np.zeros(input_frame, dtype=np.float32)
    n_frames = int(len(audio) // hop_size) + 1                                   # F0_Extractor / Volume_Extractor
    start_frame = int(silence_front * samplerate / hop_size)
    trim = int(np.round(start_frame * hop_size / samplerate * samplerate))
    u2w_start = int(silence_front * MODEL_SR / BLOCK_SIZE)                       # Unit2Wav.forward
    ddsp_wav = torch.zeros(1, n_frames * BLOCK_SIZE)[:, u2w_start * BLOCK_SIZE:]
    pad_left = (WIN - VOC_HOP) // 2                                              # nvSTFT.get_mel
    pad_right = max((WIN - VOC_HOP + 1) // 2, WIN - ddsp_wav.size(-1) - pad_left)
    y = torch.nn.functional.pad(ddsp_wav.unsqueeze(1), (pad_left, pad_right), mode="constant").squeeze(1)
    spec = torch.stft(y, WIN, hop_length=VOC_HOP, win_length=WIN, window=torch.hann_window(WIN), center=False,
                      return_complex=True)
    mel_frames = spec.shape[-1]
    output = torch.zeros(1, 1, mel_frames * VOC_HOP)                             # the vocoder: hop samples per frame
    mask = torch.arange(n_frames * BLOCK_SIZE)[None]                             # upsample(mask, block_size): samples
    first = int(mask[:, -output.shape[-1]:][0, 0])
    if MODEL_SR != samplerate:
        from torchaudio.transforms import Resample
        output = Resample(MODEL_SR, samplerate, lowpass_filter_width=128)(output.squeeze())
    idx = torch.arange(output.numel())
    temp = idx[-block_frame - crossfade_frame - sola_search_frame - last_delay_frame:-last_delay_frame]
    return dict(block=block_frame, cf=crossfade_frame, search=sola_search_frame, delay=last_delay_frame,
                n_in=input_frame, silence_front=silence_front, hop=hop_size, n_frames=n_frames,
                start_frame=start_frame, trim=trim, mel_start=u2w_start, mel_frames=mel_frames,
                out_len=mel_frames * VOC_HOP, mask_first=first, out_dev=output.numel(),
                tail=(int(temp[0]), int(temp[-1]) + 1))


@pytest.mark.parametrize("samplerate,block_time,crossfade_time,extra_time", [
    (44100, 0.5, 0.04, 2.0),                       # gui_reflow.py's Config defaults
    (44100, 0.3, 0.05, 1.0),
    (44100, 1.0, 0.04, 3.5),
    (22050, 0.4, 0.04, 2.5),
    (88200, 0.25, 0.03, 1.2),
    (44100, 0.2, 0.04, 0.35),                      # silence_front 0: the whole ring reaches the mel
])
def test_frames_follow_gui_reflow(samplerate, block_time, crossfade_time, extra_time):
    got = reflow_frames(samplerate, block_time, crossfade_time, extra_time, MODEL_SR, BLOCK_SIZE, VOC_HOP, WIN)
    want = gui_reflow(samplerate, block_time, crossfade_time, extra_time)
    for k in ("block", "cf", "search", "delay", "n_in", "silence_front", "hop", "n_frames", "start_frame", "trim",
              "mel_start", "mel_frames", "out_len", "out_dev", "tail"):
        assert got[k] == want[k], (k, got[k], want[k])
    assert got["mask_offset"] * BLOCK_SIZE == want["mask_first"]


def test_frames_at_the_gui_defaults():
    f = reflow_frames(44100, 0.5, 0.04, 2.0, MODEL_SR, BLOCK_SIZE, VOC_HOP, WIN)
    assert (f["n_frames"], f["mel_start"], f["mel_frames"], f["mask_offset"]) == (216, 163, 53, 163)


def test_frames_reject_a_non_integer_hop():
    with pytest.raises(ValueError, match="integer hop"):
        reflow_frames(48000, 0.5, 0.04, 2.0, MODEL_SR, BLOCK_SIZE, VOC_HOP, WIN)


@pytest.mark.parametrize("extra_time", [0.1, 0.5, 2.0, 4.0])
@pytest.mark.parametrize("crossfade_time", [0.01, 0.04, 0.15])
def test_the_output_covers_the_sola_window(extra_time, crossfade_time):
    assert reflow_frames(44100, 0.3, crossfade_time, extra_time, MODEL_SR, BLOCK_SIZE, VOC_HOP, WIN)["tail"][0] >= 0
