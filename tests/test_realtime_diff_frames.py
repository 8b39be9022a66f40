"""Without a GPU: the package's Unit2Mel, Unit2Wav and Unit2WavFast (ddsp_svc_b200/diffusion_vocoder.py) have the
reference's parameter trees (tests/golden/diffusion_cascade_state_dicts.json) and load them strictly, RealtimeDiffVC's
argument checks, and diff_frames (ddsp_svc_b200/realtime.py), the gui_diff.py block's frame bookkeeping, pinned against
gui_diff.py's own formulas restated here: GUI.set_values, SvcDDSP.infer's silence_front, F0_Extractor's frames and
trim, DiffGtMel.infer's start_frame with its crops and pad, nvSTFT's frames (torch.stft with its padding) and the SOLA
window of audio_callback after torchaudio's resampling."""
import json
import os

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import diffusion_vocoder as dv
from ddsp_svc_b200.realtime import RealtimeDiffVC, diff_frames
from tests.golden.make_golden_diffusion_cascade import MODELS

HERE = os.path.dirname(os.path.abspath(__file__))
MODEL_SR, BLOCK_SIZE, VOC_SR, VOC_HOP, WIN = 44100, 512, 44100, 512, 2048


@pytest.mark.parametrize("name", list(MODELS))
def test_cascade_has_the_reference_tree(name):
    with open(os.path.join(HERE, "golden", "diffusion_cascade_state_dicts.json")) as f:
        ref = json.load(f)[name]
    cls, kw = MODELS[name]
    net = getattr(dv, cls)(**kw)
    assert [[k, list(v.shape)] for k, v in net.state_dict().items()] == ref
    sd = {k: torch.full(shape, 0.5) for k, shape in ref}
    net.load_state_dict(sd, strict=True)
    den = (net.decoder if cls == "Unit2Mel" else net.diff_model).denoise_fn
    assert den.output_projection.weight.detach().eq(0.5).all()


def test_load_model_vocoder_builds_each_type_and_refuses_others():
    data = dv.DotDict(dict(sampling_rate=44100, block_size=512, encoder_out_channels=256))
    for kind, cls in (("Diffusion", dv.Unit2Mel), ("DiffusionNew", dv.Unit2Wav), ("DiffusionFast", dv.Unit2WavFast)):
        model = dv.DotDict(dict(type=kind, n_spk=1, use_pitch_aug=False, n_layers=1, n_chans=64, n_hidden=256,
                                win_length=2048))
        assert type(dv.build_model(dv.DotDict(data=data, model=model), 128)) is cls
    with pytest.raises(ValueError, match="Unknown Model"):
        dv.build_model(dv.DotDict(data=data, model=dict(type="RectifiedFlow")), 128)


def test_unit2mel_needs_a_256_wide_condition():
    with pytest.raises(ValueError, match="n_hidden"):
        dv.Unit2Mel(256, 1, n_layers=1, n_chans=64, n_hidden=384)


@pytest.mark.parametrize("cls,args", [(dv.Unit2Mel, (256, 1, False, 128, 1, 64)),
                                      (dv.Unit2Wav, (44100, 512, 256, 1, False, 128, 1, 64)),
                                      (dv.Unit2WavFast, (44100, 512, 2048, 256, 1, False, 128, 1, 64))])
def test_cascade_refuses_training(cls, args):
    with pytest.raises(NotImplementedError, match="patch_reference"):
        cls(*args)(None, None, None, infer=False)


@pytest.mark.parametrize("kw,match", [(dict(pitch_extractor_type="harvest"), "rmvpe"),
                                      (dict(diff_method="euler"), "diff_method"),
                                      (dict(k_step=-1), "k_step"), (dict(k_step=2.5), "k_step"),
                                      (dict(diff_acc=0), "diff_acc"), (dict(k_step=100, diff_acc=51), "diff_acc"),
                                      (dict(k_step=3, diff_acc=2), "diff_acc"), (dict(diff_acc=1.5), "diff_acc")])
def test_session_arguments_checked_before_loading(kw, match):
    with pytest.raises(ValueError, match=match):
        RealtimeDiffVC("no/such/ddsp.pt", "no/such/model.pt", **kw)


def gui_diff(samplerate, block_time, crossfade_time, extra_time, diff_silence):
    """gui_diff.py's own arithmetic for one block"""
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
    ddsp_out = torch.zeros(1, n_frames * BLOCK_SIZE)                             # the DDSP model's output
    f0 = torch.zeros(1, n_frames, 1)
    diff_start = int(silence_front * VOC_SR / VOC_HOP)                           # DiffGtMel.infer
    if diff_silence:
        ddsp_out = ddsp_out[:, diff_start * VOC_HOP:]
        f0 = f0[:, diff_start:, :]
        crop = 0
    else:
        crop = diff_start
    pad_left = (WIN - VOC_HOP) // 2                                              # nvSTFT.get_mel
    pad_right = max((WIN - VOC_HOP + 1) // 2, WIN - ddsp_out.size(-1) - pad_left)
    y = torch.nn.functional.pad(ddsp_out.unsqueeze(1), (pad_left, pad_right), mode="constant").squeeze(1)
    spec = torch.stft(y, WIN, hop_length=VOC_HOP, win_length=WIN, window=torch.hann_window(WIN), center=False,
                      return_complex=True)
    mel_frames = spec.shape[-1]
    out_mel = torch.zeros(1, mel_frames, 128)
    if crop > 0:                                                                 # DiffGtMel.__call__
        out_mel, f0 = out_mel[:, crop:, :], f0[:, crop:, :]
    output = torch.zeros(1, 1, out_mel.shape[1] * VOC_HOP)
    voc_frames = out_mel.shape[1]
    if crop > 0:
        output = torch.nn.functional.pad(output, (crop * VOC_HOP, 0))
    if diff_silence and diff_start > 0:
        output = torch.nn.functional.pad(output, (diff_start * VOC_HOP, 0))
    mask = torch.ones(1, n_frames * BLOCK_SIZE)
    output = output * mask                                                       # output *= mask must broadcast
    if MODEL_SR != samplerate:
        from torchaudio.transforms import Resample
        output = Resample(MODEL_SR, samplerate, lowpass_filter_width=128)(output.squeeze())
    idx = torch.arange(output.numel())
    temp = idx[-block_frame - crossfade_frame - sola_search_frame - last_delay_frame:-last_delay_frame]
    return dict(block=block_frame, cf=crossfade_frame, search=sola_search_frame, delay=last_delay_frame,
                n_in=input_frame, silence_front=silence_front, hop=hop_size, n_frames=n_frames,
                start_frame=start_frame, trim=trim, diff_start=diff_start, cond_frames=ddsp_out.shape[1] // BLOCK_SIZE,
                mel_frames=mel_frames, voc_frames=voc_frames, out_len=mask.shape[1], out_dev=output.numel(),
                tail=(int(temp[0]), int(temp[-1]) + 1))


@pytest.mark.parametrize("diff_silence", [False, True])
@pytest.mark.parametrize("samplerate,block_time,crossfade_time,extra_time", [
    (44100, 0.5, 0.04, 2.0),                       # gui_diff.py's Config defaults
    (44100, 0.3, 0.05, 1.0),
    (44100, 1.0, 0.04, 3.5),
    (22050, 0.4, 0.04, 2.5),
    (88200, 0.25, 0.03, 1.2),
    (44100, 0.2, 0.04, 0.35),                      # silence_front 0: no crop and no pad
])
def test_frames_follow_gui_diff(samplerate, block_time, crossfade_time, extra_time, diff_silence):
    got = diff_frames(samplerate, block_time, crossfade_time, extra_time, MODEL_SR, BLOCK_SIZE, VOC_SR, VOC_HOP, WIN,
                      diff_silence)
    want = gui_diff(samplerate, block_time, crossfade_time, extra_time, diff_silence)
    for k in ("block", "cf", "search", "delay", "n_in", "silence_front", "hop", "n_frames", "start_frame", "trim",
              "diff_start", "cond_frames", "mel_frames", "voc_frames", "out_len", "out_dev", "tail"):
        assert got[k] == want[k], (k, got[k], want[k])


def test_frames_at_the_gui_defaults():
    f = diff_frames(44100, 0.5, 0.04, 2.0, MODEL_SR, BLOCK_SIZE, VOC_SR, VOC_HOP, WIN)
    assert (f["n_frames"], f["diff_start"], f["cond_frames"], f["voc_frames"]) == (216, 163, 216, 53)
    f = diff_frames(44100, 0.5, 0.04, 2.0, MODEL_SR, BLOCK_SIZE, VOC_SR, VOC_HOP, WIN, diff_silence=True)
    assert (f["cond_frames"], f["mel_frames"], f["voc_frames"]) == (53, 53, 53)


@pytest.mark.parametrize("args,match", [((48000, 0.5, 0.04, 2.0, MODEL_SR, BLOCK_SIZE, VOC_SR, VOC_HOP), "integer hop"),
                                        ((44100, 0.5, 0.04, 2.0, MODEL_SR, BLOCK_SIZE, 22050, VOC_HOP), "vocoder"),
                                        ((44100, 0.5, 0.04, 2.0, MODEL_SR, BLOCK_SIZE, VOC_SR, 256), "vocoder")])
def test_frames_reject_what_the_reference_cannot_run(args, match):
    with pytest.raises(ValueError, match=match):
        diff_frames(*args)


@pytest.mark.parametrize("extra_time", [0.1, 0.5, 2.0, 4.0])
@pytest.mark.parametrize("crossfade_time", [0.01, 0.04, 0.15])
def test_the_output_covers_the_sola_window(extra_time, crossfade_time):
    for silence in (False, True):
        f = diff_frames(44100, 0.3, crossfade_time, extra_time, MODEL_SR, BLOCK_SIZE, VOC_SR, VOC_HOP, WIN, silence)
        assert f["tail"][0] >= 0
