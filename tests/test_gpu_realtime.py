"""The real-time block's kernels (csrc/realtime.cu) and ddsp_svc_b200.enhancer.Enhancer on the GPU, against the float64
oracle (tests/realtime_oracle.py) and, for the enhancer, against the reference's formulation: host np.interp and
torchaudio's Resample around the same generator, mel and noise."""
import functools
import json
import warnings

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import ops
from ddsp_svc_b200.enhancer import Enhancer
from tests import realtime_oracle as ro
from tests import hifigan_oracle as ho
from tests import report
from tests.golden import make_golden_hifigan as mk
from tests.test_realtime import CASES, f0_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _d(a, dtype=torch.float32):
    return torch.as_tensor(np.asarray(a)).to(dtype).to(DEV)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("sr,start_frame,key", [(44100, 0, 0), (44100, 7, 3), (48000, 0, -2), (48000, 13, 12)])
def test_f0_regrid_rmvpe(case, sr, start_frame, key):
    """F0_Extractor's rmvpe post-processing with uv_interp, SvcDDSP.infer's pitch factor: the GUI's 2.4 s window, and
    the silence_front frames of its default safe_prefix_pad_length"""
    f0 = f0_case(case, 241, seed=sr + start_frame)
    hop = 512 * sr / 44100
    n_frames = int(2.41 * sr // hop) + 1
    got = ops.rt_f0_regrid(_d(f0), 0.01, n_frames, hop / sr, rmvpe=True, pad=start_frame, f0_min=50.0,
                           post_scale=2 ** (key / 12)).cpu().numpy()
    ref = ro.rmvpe_f0(f0, hop, sr, n_frames, start_frame, 50.0, key)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0)
    report.record("realtime/regrid_rmvpe/%s_%d_%d" % (case, sr, start_frame),
                  max_rel=float(np.max(np.abs(got - ref) / np.maximum(ref, 1e-30))))


@pytest.mark.parametrize("key", range(8))
@pytest.mark.parametrize("start_frame", [0, 9])
def test_f0_regrid_enhancer(key, start_frame):
    f0 = ro.rmvpe_f0(f0_case("edges"), 512, 44100, 207, 0, 50.0, 0)
    rate, real = ro.adaptive_rate(44100, key)
    n_frames = int(200 * 512 * rate / 44100 // 512 + 1)
    got = ops.rt_f0_regrid(_d(f0[start_frame:]), 512 / 44100, n_frames, 512 / 44100, src_div=real,
                           src_scale=real).cpu().numpy()
    ref = ro.enhancer_f0(f0, 512, 44100, real, 512, 44100, n_frames, start_frame)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0)


def _sola_case(cf, search, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(cf + search).astype(np.float32)
    s0 = int(rng.integers(0, search + 1))
    buf = (x[s0:s0 + cf] + 0.5 * rng.standard_normal(cf)).astype(np.float32)
    return x, buf


@pytest.mark.parametrize("sr,crossfade_time", [(44100, 0.04), (48000, 0.04), (44100, 0.03), (22050, 0.07),
                                               (16000, 0.15)])
@pytest.mark.parametrize("seed", range(4))
def test_sola(sr, crossfade_time, seed):
    """the shift equals the oracle's wherever its best score beats the runner-up by more than 1e-4 relative"""
    cf, search = int(crossfade_time * sr), int(0.01 * sr)
    x, buf = _sola_case(cf, search, seed)
    scores = ro.sola_scores(x, buf, search)
    best = int(np.argmax(scores))
    runner = np.max(np.delete(scores, best)) if search else -np.inf
    got = int(ops.rt_sola(_d(x), _d(buf), search).item())
    if scores[best] - runner > 1e-4 * abs(scores[best]):
        assert got == best
    else:
        assert scores[got] >= scores[best] - 1e-4 * abs(scores[best])


@pytest.mark.parametrize("pv", [False, True])
@pytest.mark.parametrize("sr,block_time,crossfade_time", [(44100, 0.3, 0.04), (48000, 0.3, 0.04), (44100, 0.3, 0.03),
                                                          (22050, 0.05, 0.15), (16000, 1.0, 0.07)])
def test_crossfade(pv, sr, block_time, crossfade_time):
    """at the GUI defaults, 48 kHz, odd crossfade lengths (1323, 3307) and a block shorter than the crossfade"""
    block, cf, search = int(block_time * sr), int(crossfade_time * sr), int(0.01 * sr)
    rng = np.random.default_rng(block + cf)
    x = (0.3 * rng.standard_normal(block + cf + search)).astype(np.float32)
    buf = (0.3 * rng.standard_normal(cf)).astype(np.float32)
    fade_in = torch.sin(np.pi * torch.arange(0, 1, 1 / cf, device=DEV) / 2) ** 2        # start_vc's windows
    fade_out = 1 - fade_in
    shift = int(rng.integers(0, search + 1))
    xd, bufd = _d(x), _d(buf)
    out, nxt = ops.rt_crossfade(xd, torch.tensor([shift], dtype=torch.int32, device=DEV), search, bufd, fade_in,
                                fade_out, block, pv)
    got = torch.cat([out, nxt]).cpu().double().numpy()
    if pv:
        ref = np.concatenate(ro.crossfade(x, shift, buf, fade_in.cpu().numpy(), fade_out.cpu().numpy(), block, True))
        err = np.abs(got - ref).max() / np.abs(ref).max()
        report.record("realtime/pv/%d_%d" % (sr, cf), rel_max=err)
        assert err < 2e-5, err
    else:
        temp = xd[shift:shift + block + cf].clone()                  # gui.py's fp32 lines
        temp[:cf] *= fade_in
        temp[:cf] += bufd * fade_out
        assert torch.equal(torch.cat([out, nxt]), temp)


def test_shift_from_sola_feeds_crossfade_without_sync_and_replays_in_a_graph():
    sr, block, cf, search = 44100, 13230, 1764, 441
    rng = np.random.default_rng(5)
    x = _d(0.3 * rng.standard_normal(block + cf + search))
    buf = _d(0.3 * rng.standard_normal(cf))
    f0 = _d(f0_case("voiced"))
    fade_in = torch.sin(np.pi * torch.arange(0, 1, 1 / cf, device=DEV) / 2) ** 2
    fade_out = 1 - fade_in

    def block_fn():
        g = ops.rt_f0_regrid(f0, 0.01, 208, 512 / 44100, rmvpe=True, pad=3, f0_min=50.0, post_scale=1.5)
        shift = ops.rt_sola(x, buf, search)
        return (g,) + ops.rt_crossfade(x, shift, search, buf, fade_in, fade_out, block, True)

    eager = block_fn()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = block_fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for a, b in zip(eager, again):
        assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        block_fn()                                                   # warm the allocator on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = block_fn()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, static):
        assert torch.equal(a, b)


# ---- Enhancer ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def enhancer_ckpt(tmp_path_factory):
    d = tmp_path_factory.mktemp("enhancer")
    cfg = dict(ho.SMALL, sampling_rate=44100, num_mels=128, n_fft=2048, win_size=2048, hop_size=512, fmin=40,
               fmax=16000)
    (d / "config.json").write_text(json.dumps(cfg))
    torch.save({"generator": mk.seeded_state_dict("small")}, str(d / "model.ckpt"))
    return str(d / "model.ckpt")


@pytest.fixture(scope="module")
def enhancer(enhancer_ckpt):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        enh = Enhancer("nsf-hifigan", enhancer_ckpt, device=DEV)
    g = torch.Generator().manual_seed(3)
    noise_ = torch.randn(1, 600 * 512, 9, generator=g).to(DEV)
    rand_ini = torch.rand(1, 1, 9, generator=g)
    rand_ini[..., 0] = 0
    forward = functools.partial(type(enh.model).forward, enh.model, rand_ini=rand_ini.to(DEV))
    # the same draws for both arms: noise cut to each call's length
    enh.model.forward = lambda x, f0, rand_ini=None, noise=None: forward(x, f0, noise=noise_[:, :x.shape[-1] * 512].contiguous())
    return enh


def reference_enhance(enh, audio, sample_rate, f0, hop_size, adaptive_key, silence_front):
    """enhancer.py:23-85 restated with the package's generator and mel: host np.interp, torchaudio Resample"""
    from torchaudio.transforms import Resample
    esr, ehop = enh.enhancer_sample_rate, enh.enhancer_hop_size
    start_frame = int(silence_front * sample_rate / hop_size)
    real_silence_front = start_frame * hop_size / sample_rate
    audio = audio[:, int(np.round(real_silence_front * sample_rate)):]
    f0 = f0[:, start_frame:, :]
    if adaptive_key == 'auto':
        adaptive_key = max(0, np.ceil(12 * np.log2(float(torch.max(f0) / 760))))
    rate, real = ro.adaptive_rate(esr, adaptive_key)
    audio_res = audio if sample_rate == rate else Resample(sample_rate, rate, lowpass_filter_width=128).to(DEV)(audio)
    n_frames = int(audio_res.size(-1) // ehop + 1)
    f0_np = f0.squeeze(0).squeeze(-1).cpu().numpy()
    f0_np *= real
    f0_res = np.interp((ehop / esr) * np.arange(n_frames), (hop_size / sample_rate) * np.arange(len(f0_np)) / real,
                       f0_np, left=f0_np[0], right=f0_np[-1])
    f0_res = torch.from_numpy(f0_res).unsqueeze(0).float().to(DEV)
    with torch.no_grad():
        mel = enh.stft.get_mel(audio_res)
        out = enh.model(mel, f0_res[:, :mel.size(-1)])
    if rate != esr:
        out = Resample(rate, esr, lowpass_filter_width=128).to(DEV)(out)
    if start_frame > 0:
        out = torch.nn.functional.pad(out, (int(np.round(esr * real_silence_front)), 0))
    return out, esr


@pytest.mark.parametrize("key", list(range(8)) + ["auto"])
@pytest.mark.parametrize("silence_front", [0.0, 0.07])
def test_enhancer_matches_the_reference_formulation(enhancer, key, silence_front):
    rng = np.random.default_rng(11)
    n = 44100
    t = np.arange(n) / 44100
    f0_frames = 200 + 40 * np.sin(2 * np.pi * np.arange(n // 512 + 1) / 50)
    audio = _d(0.3 * np.sin(2 * np.pi * np.cumsum(np.repeat(f0_frames, 512)[:n]) / 44100)
               + 0.01 * rng.standard_normal(n))[None]
    f0 = _d(f0_frames)[None, :, None]
    if key == "auto":
        f0 = f0 * 4                                                  # max 960 Hz: 'auto' picks key 5
    got, sr = enhancer.enhance(audio, 44100, f0, 512, adaptive_key=key, silence_front=silence_front)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):   # torchaudio's convolution in plain fp32
        ref, rsr = reference_enhance(enhancer, audio, 44100, f0, 512, key, silence_front)
    assert sr == rsr == 44100 and got.shape == ref.shape, (got.shape, ref.shape)
    rel = ((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    report.record("realtime/enhancer/%s_%g" % (key, silence_front), rel_rms=rel)
    assert rel < 1e-4, rel


def test_enhancer_numeric_key_does_not_sync(enhancer):
    audio = _d(0.1 * np.random.default_rng(1).standard_normal((1, 30000)))
    f0 = _d(np.full((1, 59, 1), 220.0))
    enhancer.enhance(audio, 44100, f0, 512, adaptive_key=2)         # builds the resampling tables
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        enhancer.enhance(audio, 44100, f0, 512, adaptive_key=2)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_enhancer_rejects_unknown_type(enhancer_ckpt):
    with pytest.raises(ValueError, match="Unknown enhancer"):
        Enhancer("nsf-hifigan-x", enhancer_ckpt, device=DEV)
