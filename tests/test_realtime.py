"""The real-time block's kernels (csrc/realtime.cu) without a GPU: the float64 oracle (tests/realtime_oracle.py) against
np.interp, np.fft.rfft and np.correlate; the kernels' source run on the CPU (tests/emu/emu_realtime.cpp) against the
oracle, under ThreadSanitizer, and the C ABI's argument checks.  The kernels run on hardware in
tests/test_gpu_realtime.py."""
import ctypes

import numpy as np
import pytest
import torch

from tests import realtime_oracle as ro
from tests.emu_harness import abi_call, assert_race_free, shared, tsan

HOP = 512 * 44100 / 44100                       # SvcDDSP.infer's hop_size for block_size 512 at the model's rate


def f0_case(name, n=241, seed=0):
    """10 ms RMVPE-like f0 (float32, 0 = unvoiced)"""
    rng = np.random.default_rng(seed)
    f = (220 * 2 ** (rng.standard_normal(n) * 0.3)).astype(np.float32)
    if name == "voiced":
        f[rng.random(n) < 0.3] = 0
    elif name == "unvoiced":
        f[:] = 0
    elif name == "single":
        f[np.arange(n) != n // 3] = 0
    elif name == "edges":
        f[3:-4] = 0
    return f


CASES = ["voiced", "unvoiced", "single", "edges"]


# ---- the oracle against independent formulations ----------------------------------------------------------------------
def test_interp_matches_numpy():
    rng = np.random.default_rng(1)
    xp = 0.01 * np.arange(57)
    fp = rng.standard_normal(57)
    x = np.concatenate([512 / 44100 * np.arange(60), [0.0, xp[-1], xp[10], 1.0]])
    assert np.array_equal(ro.interp(x, xp, fp), np.interp(x, xp, fp))


@pytest.mark.parametrize("case", CASES)
def test_fill_matches_numpy(case):
    f = f0_case(case)
    ref = f.copy()
    uv = ref == 0
    if len(ref[~uv]) > 0:
        ref[uv] = np.interp(np.where(uv)[0], np.where(~uv)[0], ref[~uv])
    assert np.array_equal(ro.fill_unvoiced(f), ref)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("start_frame", [0, 9])
def test_rmvpe_f0_matches_numpy(case, start_frame):
    f0 = f0_case(case)
    n_frames, f0_min, key = 200, 50.0, 3.0
    f = f0.copy()
    uv = f == 0
    if len(f[~uv]) > 0:
        f[uv] = np.interp(np.where(uv)[0], np.where(~uv)[0], f[~uv])
    src, dst = 0.01 * np.arange(len(f)), HOP / 44100 * np.arange(n_frames - start_frame)
    g = np.interp(dst, src, f)
    g[np.interp(dst, src, uv.astype(float)) > 0.5] = 0
    g = np.pad(g, (start_frame, 0))
    uv = g == 0
    if len(g[~uv]) > 0:
        g[uv] = np.interp(np.where(uv)[0], np.where(~uv)[0], g[~uv])
    g[g < f0_min] = f0_min
    ref = (torch.from_numpy(g).float() * 2 ** (key / 12)).numpy()
    assert np.array_equal(ro.rmvpe_f0(f0, HOP, 44100, n_frames, start_frame, f0_min, key), ref)


@pytest.mark.parametrize("key", [0, 3, 7])
def test_enhancer_f0_matches_numpy(key):
    f0 = f0_case("voiced")
    f0[f0 == 0] = 150
    rate, real = ro.adaptive_rate(44100, key)
    n_frames = 300
    f = f0.copy()
    f *= real
    ref = np.interp(512 / 44100 * np.arange(n_frames), (HOP / 44100) * np.arange(len(f)) / real, f, left=f[0],
                    right=f[-1]).astype(np.float32)
    assert np.array_equal(ro.enhancer_f0(f0, HOP, 44100, real, 512, 44100, n_frames), ref)


def test_sola_matches_correlate():
    rng = np.random.default_rng(2)
    x, buf = rng.standard_normal(1764 + 441), rng.standard_normal(1764)
    nom = np.correlate(x, buf, "valid")
    den = np.sqrt(np.correlate(x ** 2, np.ones(1764), "valid") + 1e-8)
    np.testing.assert_allclose(ro.sola_scores(x, buf, 441), nom / den, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("n", [1764, 441, 1323])
def test_phase_vocoder_matches_rfft(n):
    rng = np.random.default_rng(n)
    a, b = rng.standard_normal(n), rng.standard_normal(n)
    fade_in, fade_out = ro.fade_windows(n)
    w = np.sqrt(fade_out * fade_in)
    fa, fb = np.fft.rfft(a * w), np.fft.rfft(b * w)
    absab = np.abs(fa) + np.abs(fb)
    absab[1:-1 if n % 2 == 0 else None] *= 2
    d = np.angle(fb) - np.angle(fa)
    d = d - 2 * np.pi * np.floor(d / 2 / np.pi + 0.5)
    wk = 2 * np.pi * np.arange(n // 2 + 1) + d
    t = np.arange(n)[:, None] / n
    ref = a * fade_out ** 2 + b * fade_in ** 2 + np.sum(absab * np.cos(wk * t + np.angle(fa)), -1) * w / n
    np.testing.assert_allclose(ro.phase_vocoder(a, b, fade_out, fade_in), ref, rtol=0, atol=1e-9)


@pytest.mark.parametrize("sr", [16000, 22050, 44100, 48000])
@pytest.mark.parametrize("crossfade_time", [0.01, 0.04, 0.07, 0.15])
def test_fade_window_length(sr, crossfade_time):
    """start_vc's torch.arange(0, 1, 1 / crossfade) has exactly crossfade elements at the GUI's rates and lengths"""
    cf = int(crossfade_time * sr)
    assert torch.arange(0, 1, 1 / cf).numel() == cf


# ---- the kernels' source on the CPU --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return shared("emu_realtime.cpp", tmp_path_factory)


def _p(a):
    return a.ctypes.data


def run_regrid(emu, src, src_step, n_dst, dst_step, src_div=1.0, src_scale=1.0, mode=0, pad=0, f0_min=0.0,
               post_scale=1.0):
    src = np.ascontiguousarray(src, np.float32)
    out = np.full(n_dst, np.nan, np.float32)
    vsrc, vdst = np.empty(len(src)), np.empty(n_dst)
    prev = np.empty(max(len(src), n_dst), np.int32)
    emu.emu_rt_f0_regrid(_p(src), len(src), src_step, src_div, src_scale, n_dst, pad, dst_step, mode, f0_min,
                         post_scale, _p(out), _p(vsrc), _p(vdst), _p(prev))
    return out


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("sr,start_frame,n10", [(44100, 0, 241), (48000, 13, 241), (44100, 5, 700)])
def test_emu_regrid_rmvpe(emu, case, sr, start_frame, n10):
    """F0_Extractor's post-processing: 700 source frames run the neighbour scans over three chunks"""
    f0 = f0_case(case, n10, seed=n10)
    hop = 512 * sr / 44100
    n_frames = int(n10 * 0.01 * sr // hop)
    got = run_regrid(emu, f0, 0.01, n_frames, hop / sr, mode=1, pad=start_frame, f0_min=50.0,
                     post_scale=2 ** (5 / 12))
    ref = ro.rmvpe_f0(f0, hop, sr, n_frames, start_frame, 50.0, 5)
    np.testing.assert_array_equal(got, ref)


@pytest.mark.parametrize("key", [0, 1, 4, 7])
@pytest.mark.parametrize("start_frame", [0, 11])
def test_emu_regrid_enhancer(emu, key, start_frame):
    f0 = ro.rmvpe_f0(f0_case("voiced"), HOP, 44100, 200, 0, 50.0)
    rate, real = ro.adaptive_rate(44100, key)
    n_frames = 250
    got = run_regrid(emu, f0[start_frame:], HOP / 44100, n_frames, 512 / 44100, src_div=real, src_scale=real)
    np.testing.assert_array_equal(got, ro.enhancer_f0(f0, HOP, 44100, real, 512, 44100, n_frames, start_frame))


def _sola_case(cf, search, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(cf + search).astype(np.float32)
    s0 = int(rng.integers(0, search + 1))
    buf = (x[s0:s0 + cf] + 0.3 * rng.standard_normal(cf)).astype(np.float32)
    return x, buf


@pytest.mark.parametrize("cf,search", [(1764, 441), (480, 480), (300, 5), (1323, 0)])
def test_emu_sola(emu, cf, search):
    x, buf = _sola_case(cf, search, cf)
    shift = np.full(1, -1, np.int32)
    emu.emu_rt_sola(_p(x), _p(buf), cf, search, _p(shift))
    assert shift[0] == int(np.argmax(ro.sola_scores(x, buf, search)))


def fade_windows32(cf):
    """the windows as start_vc builds them (fp32 torch)"""
    fade_in = torch.sin(np.pi * torch.arange(0, 1, 1 / cf) / 2) ** 2
    return fade_in.numpy(), (1 - fade_in).numpy()


@pytest.mark.parametrize("pv", [False, True])
@pytest.mark.parametrize("block,cf,shift", [(1000, 441, 17), (300, 441, 3), (2000, 1323, 0)])
def test_emu_crossfade(emu, pv, block, cf, shift):
    """the fade at a shift read from memory; block < crossfade puts faded samples into the next SOLA buffer"""
    rng = np.random.default_rng(block + cf)
    x = rng.standard_normal(block + cf + 40).astype(np.float32)
    buf = rng.standard_normal(cf).astype(np.float32)
    fade_in, fade_out = fade_windows32(cf)
    out, nxt = np.full(block, np.nan, np.float32), np.full(cf, np.nan, np.float32)
    bins = np.full(3 * (cf // 2 + 1), np.nan, np.float32)
    sh = np.array([shift], np.int32)
    emu.emu_rt_crossfade(_p(x), _p(sh), _p(buf), _p(fade_in), _p(fade_out), block, cf, int(pv), _p(out), _p(nxt),
                         _p(bins))
    ref_out, ref_next = ro.crossfade(x, shift, buf, fade_in, fade_out, block, pv)
    got = np.concatenate([out, nxt])
    ref = np.concatenate([ref_out, ref_next])
    if pv:
        np.testing.assert_allclose(got, ref, rtol=0, atol=2e-5 * np.abs(ref).max())
    else:
        x32 = x[shift:shift + block + cf].copy()
        x32[:cf] = x32[:cf] * fade_in + buf * fade_out               # the reference's fp32 order
        np.testing.assert_array_equal(got, x32)


def test_tsan_realtime(tmp_path):
    assert_race_free(tsan("tsan_realtime.cpp", tmp_path))


# ---- C ABI argument checks (no CUDA call is made) -------------------------------------------------------------------
def test_abi_errors():
    base = dict(src=8, n_src=10, src_step=0.01, src_div=1.0, src_scale=1.0, n_dst=10, pad=0, dst_step=0.01, mode=1,
                f0_min=50.0, post_scale=1.0, out=8, workspace=16, workspace_bytes=1 << 20, stream=None)
    assert abi_call("b2d_rt_f0_regrid", dict(base, src=None)) == -1
    assert abi_call("b2d_rt_f0_regrid", dict(base, pad=11)) == -2
    assert abi_call("b2d_rt_f0_regrid", dict(base, mode=0, pad=1)) == -2
    assert abi_call("b2d_rt_f0_regrid", dict(base, workspace_bytes=64)) == -5
    assert abi_call("b2d_rt_sola", dict(x=8, buf=8, crossfade=0, search=1, shift=8, stream=None)) == -2
    cf = dict(x=8, shift=8, buf=8, fade_in=8, fade_out=8, block=10, crossfade=40000, phase_vocoder=1, out=8,
              next_buf=8, workspace=16, workspace_bytes=1 << 20, stream=None)
    assert abi_call("b2d_rt_crossfade", cf) == -4
    assert abi_call("b2d_rt_crossfade", dict(cf, crossfade=100, workspace_bytes=4)) == -5
    assert abi_call("b2d_rt_crossfade_workspace_bytes", dict(crossfade=1764, phase_vocoder=1)) == 3 * 883 * 4
    assert isinstance(ctypes.c_size_t(abi_call("b2d_rt_f0_regrid_workspace_bytes", dict(n_src=3, n_dst=4))).value, int)
