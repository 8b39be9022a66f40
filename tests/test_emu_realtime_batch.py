"""The batched real-time block kernels (csrc/realtime.cu: b2d_rt_f0_regrid_batch, b2d_rt_sola_batch,
b2d_rt_crossfade_batch) without a GPU: their source run on the CPU (tests/emu/emu_realtime_batch.cpp) row by row
against the float64 oracle (tests/realtime_oracle.py) and bit for bit against the single-session launch
(tests/emu/emu_realtime.cpp) on the same row, on ragged batches (all-unvoiced rows, SOLA peaks at 0 and at `search`,
N = 1 and N = 5); under AddressSanitizer and ThreadSanitizer; and the C ABI's argument checks.  The kernels run on
hardware in tests/test_gpu_realtime_batch.py."""
import ctypes

import numpy as np
import pytest

from tests import realtime_oracle as ro
from tests.emu_harness import abi_call, asan, assert_race_free, shared, tsan
from tests.test_realtime import HOP, f0_case, fade_windows32, run_regrid

ROW_CASES = ["voiced", "unvoiced", "single", "edges", "voiced"]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return shared("emu_realtime_batch.cpp", tmp_path_factory)


@pytest.fixture(scope="module")
def emu1(tmp_path_factory):
    return shared("emu_realtime.cpp", tmp_path_factory)


def _p(a):
    return a.ctypes.data


def run_regrid_batch(emu, src, src_step, n_dst, dst_step, src_div=1.0, src_scale=1.0, mode=0, pad=0, f0_min=0.0,
                     post_scale=None):
    src = np.ascontiguousarray(src, np.float32)
    rows, n_src = src.shape
    out = np.full((rows, n_dst), np.nan, np.float32)
    ws = np.full(rows * emu.emu_rt_regrid_row_bytes(n_src, n_dst), 0xFF, np.uint8)
    post = np.ascontiguousarray(np.ones(rows) if post_scale is None else post_scale, np.float32)
    emu.emu_rt_f0_regrid_batch(_p(src), rows, n_src, src_step, src_div, src_scale, n_dst, pad, dst_step, mode, f0_min,
                               _p(post), _p(out), _p(ws))
    return out


@pytest.mark.parametrize("rows", [1, 5])
@pytest.mark.parametrize("sr,start_frame,n10", [(44100, 0, 241), (48000, 13, 241), (44100, 5, 700)])
def test_regrid_rmvpe_rows(emu, emu1, rows, sr, start_frame, n10):
    """F0_Extractor's post-processing per row, each row with its own pitch factor; row 1 is all unvoiced"""
    f0 = np.stack([f0_case(ROW_CASES[i], n10, seed=n10 + i) for i in range(rows)])
    keys = np.array([5, -7, 0, 12, 3][:rows], np.float64)
    post = (2 ** (keys / 12)).astype(np.float32)
    hop = 512 * sr / 44100
    n_frames = int(n10 * 0.01 * sr // hop)
    got = run_regrid_batch(emu, f0, 0.01, n_frames, hop / sr, mode=1, pad=start_frame, f0_min=50.0, post_scale=post)
    for i in range(rows):
        np.testing.assert_array_equal(got[i], ro.rmvpe_f0(f0[i], hop, sr, n_frames, start_frame, 50.0, keys[i]))
        single = run_regrid(emu1, f0[i], 0.01, n_frames, hop / sr, mode=1, pad=start_frame, f0_min=50.0,
                            post_scale=float(post[i]))
        assert got[i].tobytes() == single.tobytes(), i


@pytest.mark.parametrize("rows", [1, 5])
@pytest.mark.parametrize("key", [0, 3])
def test_regrid_enhancer_rows(emu, emu1, rows, key):
    """mode 0 (Enhancer.enhance's f0 at a numeric key) for every row; post_scale is not read"""
    f0 = np.stack([ro.rmvpe_f0(f0_case(ROW_CASES[i], seed=i), HOP, 44100, 200, 0, 50.0) for i in range(rows)])
    rate, real = ro.adaptive_rate(44100, key)
    got = run_regrid_batch(emu, f0, HOP / 44100, 250, 512 / 44100, src_div=real, src_scale=real,
                           post_scale=np.full(rows, np.nan))
    for i in range(rows):
        np.testing.assert_array_equal(got[i], ro.enhancer_f0(f0[i], HOP, 44100, real, 512, 44100, 250))
        single = run_regrid(emu1, f0[i], HOP / 44100, 250, 512 / 44100, src_div=real, src_scale=real)
        assert got[i].tobytes() == single.tobytes(), i


def sola_rows(rows, cf, search, stride, peaks, seed):
    """x [rows, stride] whose row i correlates best with buf row i at shift peaks[i]"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((rows, stride)).astype(np.float32)
    buf = np.stack([x[i, p:p + cf] + 0.3 * rng.standard_normal(cf) for i, p in enumerate(peaks)]).astype(np.float32)
    return x, buf


@pytest.mark.parametrize("cf,search", [(1764, 441), (300, 5), (480, 0)])
def test_sola_rows(emu, emu1, cf, search):
    """five rows with the peak at 0, at search and between; x rows padded past cf + search (a row stride)"""
    peaks = [0, search, search // 2, 0, search]
    stride = cf + search + 17
    x, buf = sola_rows(5, cf, search, stride, peaks, cf + search)
    shift = np.full(5, -1, np.int32)
    emu.emu_rt_sola_batch(_p(x), stride, _p(buf), 5, cf, search, _p(shift))
    for i in range(5):
        want = int(np.argmax(ro.sola_scores(x[i, :cf + search], buf[i], search)))
        assert want == peaks[i] and shift[i] == want, (i, shift[i], want)
        one = np.full(1, -1, np.int32)
        emu1.emu_rt_sola(_p(np.ascontiguousarray(x[i])), _p(np.ascontiguousarray(buf[i])), cf, search, _p(one))
        assert one[0] == shift[i]


def test_sola_single_row(emu):
    x, buf = sola_rows(1, 441, 100, 541, [37], 3)
    shift = np.full(1, -1, np.int32)
    emu.emu_rt_sola_batch(_p(x), 541, _p(buf), 1, 441, 100, _p(shift))
    assert shift[0] == 37


@pytest.mark.parametrize("pv", [False, True])
@pytest.mark.parametrize("rows,block,cf,search", [(1, 1000, 441, 40), (5, 300, 441, 40), (5, 2000, 1323, 0)])
def test_crossfade_rows(emu, emu1, pv, rows, block, cf, search):
    """every row at its own shift (0, search and between), its own buffer and output row"""
    rng = np.random.default_rng(block + cf + rows)
    stride = search + block + cf + 3
    x = rng.standard_normal((rows, stride)).astype(np.float32)
    buf = rng.standard_normal((rows, cf)).astype(np.float32)
    shift = np.array([0, search, search // 3, search, 0][:rows], np.int32)
    fade_in, fade_out = fade_windows32(cf)
    out = np.full((rows, block), np.nan, np.float32)
    nxt = np.full((rows, cf), np.nan, np.float32)
    bins = np.full(rows * 3 * (cf // 2 + 1), np.nan, np.float32)
    emu.emu_rt_crossfade_batch(_p(x), stride, _p(shift), _p(buf), rows, _p(fade_in), _p(fade_out), block, cf, int(pv),
                               _p(out), _p(nxt), _p(bins))
    for i in range(rows):
        ref_out, ref_next = ro.crossfade(x[i], shift[i], buf[i], fade_in, fade_out, block, pv)
        got, ref = np.concatenate([out[i], nxt[i]]), np.concatenate([ref_out, ref_next])
        np.testing.assert_allclose(got, ref, rtol=0, atol=2e-5 * np.abs(ref).max())
        o1, n1 = np.full(block, np.nan, np.float32), np.full(cf, np.nan, np.float32)
        b1 = np.full(3 * (cf // 2 + 1), np.nan, np.float32)
        emu1.emu_rt_crossfade(_p(np.ascontiguousarray(x[i])), _p(shift[i:i + 1].copy()),
                              _p(np.ascontiguousarray(buf[i])), _p(fade_in), _p(fade_out), block, cf, int(pv), _p(o1),
                              _p(n1), _p(b1))
        assert out[i].tobytes() == o1.tobytes() and nxt[i].tobytes() == n1.tobytes(), i


def test_rows_are_independent(emu):
    """changing row 2's inputs leaves every other row's regrid, shift and crossfade bit-identical"""
    rows, cf, search, block = 5, 441, 40, 300
    f0 = np.stack([f0_case(ROW_CASES[i], seed=i) for i in range(rows)])
    post = np.array([1.0, 1.5, 0.5, 2.0, 1.25], np.float32)
    stride = search + block + cf
    x, buf = sola_rows(rows, cf, search, stride, [0, 40, 20, 7, 33], 9)
    fade_in, fade_out = fade_windows32(cf)

    def run(f0, post, x, buf):
        g = run_regrid_batch(emu, f0, 0.01, 180, HOP / 44100, mode=1, pad=4, f0_min=50.0, post_scale=post)
        shift = np.full(rows, -1, np.int32)
        emu.emu_rt_sola_batch(_p(x), stride, _p(buf), rows, cf, search, _p(shift))
        out, nxt = np.empty((rows, block), np.float32), np.empty((rows, cf), np.float32)
        bins = np.empty(rows * 3 * (cf // 2 + 1), np.float32)
        emu.emu_rt_crossfade_batch(_p(x), stride, _p(shift), _p(buf), rows, _p(fade_in), _p(fade_out), block, cf, 1,
                                   _p(out), _p(nxt), _p(bins))
        return g, shift, out, nxt

    a = run(f0, post, x, buf)
    f0b, postb, xb, bufb = f0.copy(), post.copy(), x.copy(), buf.copy()
    f0b[2] = f0_case("voiced", seed=77)
    postb[2] = 3.0
    xb[2] = np.random.default_rng(1).standard_normal(stride)
    bufb[2] = 0
    b = run(f0b, postb, xb, bufb)
    keep = [0, 1, 3, 4]
    for u, v in zip(a, b):
        assert u[keep].tobytes() == v[keep].tobytes()
    assert a[0][2].tobytes() != b[0][2].tobytes()


def test_asan_realtime_batch(tmp_path):
    """every row of every input and output in a heap buffer of exactly its size: regrid in both modes, SOLA and both
    crossfades with the last row's shift at search"""
    res = asan("emu_realtime_batch.cpp", tmp_path, "EMU_ASAN")
    assert res.returncode == 0 and "done 0" in res.stdout, res.stderr[-4000:]


def test_tsan_realtime_batch(tmp_path):
    assert_race_free(tsan("tsan_realtime_batch.cpp", tmp_path))


# ---- C ABI argument checks (no CUDA call is made) -------------------------------------------------------------------
def test_batch_abi_errors():
    base = dict(src=8, rows=3, n_src=10, src_step=0.01, src_div=1.0, src_scale=1.0, n_dst=10, pad=0, dst_step=0.01,
                mode=1, f0_min=50.0, post_scale=8, out=8, workspace=16, workspace_bytes=1 << 20, stream=None)
    row_bytes = ctypes.c_size_t(abi_call("b2d_rt_f0_regrid_workspace_bytes", dict(n_src=10, n_dst=10))).value
    assert abi_call("b2d_rt_f0_regrid_batch", dict(base, src=None)) == -1
    assert abi_call("b2d_rt_f0_regrid_batch", dict(base, post_scale=None)) == -1
    assert abi_call("b2d_rt_f0_regrid_batch", dict(base, rows=0)) == -2
    assert abi_call("b2d_rt_f0_regrid_batch", dict(base, pad=11)) == -2
    assert abi_call("b2d_rt_f0_regrid_batch", dict(base, workspace_bytes=3 * row_bytes - 1)) == -5
    assert abi_call("b2d_rt_sola_batch", dict(x=8, x_stride=100, buf=8, rows=0, crossfade=10, search=1, shift=8,
                                              stream=None)) == -2
    assert abi_call("b2d_rt_sola_batch", dict(x=8, x_stride=-1, buf=8, rows=2, crossfade=10, search=1, shift=8,
                                              stream=None)) == -2
    assert abi_call("b2d_rt_sola_batch", dict(x=8, x_stride=100, buf=None, rows=2, crossfade=10, search=1, shift=8,
                                              stream=None)) == -1
    cf = dict(x=8, x_stride=1000, shift=8, buf=8, rows=2, fade_in=8, fade_out=8, block=10, crossfade=100,
              phase_vocoder=1, out=8, next_buf=8, workspace=16, workspace_bytes=1 << 20, stream=None)
    one = ctypes.c_size_t(abi_call("b2d_rt_crossfade_workspace_bytes", dict(crossfade=100, phase_vocoder=1))).value
    assert abi_call("b2d_rt_crossfade_batch", dict(cf, crossfade=40000)) == -4
    assert abi_call("b2d_rt_crossfade_batch", dict(cf, rows=70000)) == -4
    assert abi_call("b2d_rt_crossfade_batch", dict(cf, rows=0)) == -2
    assert abi_call("b2d_rt_crossfade_batch", dict(cf, workspace_bytes=2 * one - 4)) == -5
    assert abi_call("b2d_rt_crossfade_batch", dict(cf, shift=None)) == -1
    assert abi_call("b2d_volume_mask_rows", dict(volume=8, B=2, n_frames=10, thresholds=None, mask_frames=8,
                                                 stream=None)) == -1
    assert abi_call("b2d_volume_mask_rows", dict(volume=8, B=0, n_frames=10, thresholds=8, mask_frames=8,
                                                 stream=None)) == -2
