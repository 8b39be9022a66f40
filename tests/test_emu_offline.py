"""The offline assembly's kernels (csrc/frontend.cu: slicer_rms, segment_place and cross_fade, which share the fade)
run in the CPU emulator (tests/emu/emu_offline.cpp) against float64 restatements: librosa.feature.rms's framing
(tests/offline_oracle.rms64) and main.py's cross_fade (oracle/frontend.py)."""
import numpy as np
import pytest

from oracle import frontend as fe
from tests import offline_oracle as oo
from tests.emu_harness import shared


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return shared("emu_offline.cpp", tmp_path_factory)


def ptr(a):
    return a.ctypes.data


@pytest.mark.parametrize("n,win,hop", [(44100 * 3 + 17, 3528, 882), (16000 + 5, 1280, 320), (700, 3528, 882),
                                       (1, 8, 2), (999, 7, 3), (100, 64, 1)])
def test_slicer_rms_against_float64(emu, n, win, hop):
    g = np.random.default_rng(n)
    y = (g.standard_normal(n) * np.exp(g.uniform(-8, 0, n))).astype(np.float32)
    want = oo.rms64(y, win, hop)[0]
    got = np.full(want.shape[0] + 1, np.nan, np.float32)            # one sentinel past the last frame
    assert emu.emu_slicer_rms(ptr(y), n, win, hop, ptr(got)) == 0
    assert np.isnan(got[-1])
    exact = np.sqrt(np.mean(np.pad(y.astype(np.float64), win // 2)[np.arange(win)[None] + hop * np.arange(want.shape[0])[:, None]] ** 2, 1))
    assert np.max(np.abs(got[:-1] - exact) / np.maximum(exact, 1e-30)) < 1e-6
    assert np.array_equal(got[:-1], want)                             # fp64 sums of the same terms round alike here


@pytest.mark.parametrize("seg_len,idx,fade,grid", [(1000, 300, 200, 4), (1000, 300, 200, 1), (513, 0, 0, 2),
                                                   (50, 10, 50, 1), (64, 7, 1, 1), (2000, 1999, 2, 3)])
def test_segment_place_against_main_py(emu, seg_len, idx, fade, grid):
    g = np.random.default_rng(seg_len + idx)
    result = np.zeros(idx + seg_len + 37, np.float32)
    result[:idx] = g.standard_normal(idx)
    seg = g.standard_normal(seg_len).astype(np.float32)
    before = result.copy()
    assert emu.emu_segment_place(ptr(result), ptr(seg), seg_len, idx, fade, grid) == 0
    # main.py: a = the result so far (idx + fade samples), cross_fade(a, seg, idx) in float64
    a = before[:idx + fade].astype(np.float64)
    want = fe.cross_fade(a, seg, idx) if fade else np.concatenate([a, seg])
    assert np.array_equal(result[:idx + seg_len], want.astype(np.float32))
    assert np.array_equal(result[idx + seg_len:], before[idx + seg_len:])   # nothing written past the segment


@pytest.mark.parametrize("len_a,len_b,idx,grid", [(5000, 7000, 3000, 2), (5000, 7000, 4999, 1), (300, 300, 0, 3)])
def test_cross_fade_keeps_its_fade(emu, len_a, len_b, idx, grid):
    g = np.random.default_rng(len_a + idx)
    a = g.standard_normal(len_a).astype(np.float32)
    b = g.standard_normal(len_b).astype(np.float32)
    out = np.empty(idx + len_b, np.float32)
    assert emu.emu_cross_fade(ptr(a), len_a, ptr(b), len_b, idx, ptr(out), grid) == 0
    assert np.array_equal(out, fe.cross_fade(a, b, idx).astype(np.float32))
