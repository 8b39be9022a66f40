"""csrc/mel.cu's BACKWARD kernel source executed on the CPU (tests/emu/host_emu.h) against the reference's autograd
gradients (tests/golden/mel_grad_*.npz) and the float64 restatement, race-checked under ThreadSanitizer, plus the
argument checks of its C ABI entry (no device touched).  The kernel itself runs on hardware in
tests/test_gpu_mel_backward.py."""
import ctypes

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib
from ddsp_svc_b200 import mel as pm
from tests import mel_grad_closed_form as CF
from tests import util
from tests.emu_harness import abi_call, assert_race_free, shared, tsan
from tests.golden import make_golden_mel_grad as GG

f32 = np.float32
# error model (see tests/test_gpu_mel_backward.py): the kernel's relative RMS error against float64 is at most RATIO
# times the fp32 reference's own error on the same case (emulated: 1.0 .. 1.6x)
RATIO = 3.0


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_mel_bwd.cpp", tmp_path_factory)
    basis = pm.mel_filterbank(44100, 2048, 128, 40, 16000)
    tabs = dict(basis=basis, lohi=pm._support(basis), bins=pm._bin_filters(basis),
                window=torch.hann_window(2048).numpy())
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)

    class Emu:
        def backward(self, y, hop, g, chunk):
            """g: any strided float32 array of shape [B, 128, n_frames] (read through its strides)"""
            y = np.ascontiguousarray(y, f32)
            assert g.dtype == f32
            out = np.full(y.shape, np.nan, f32)
            rc = lib.emu_mel_bwd(ptr(y), ptr(tabs["window"]), ptr(basis), ptr(tabs["lohi"]), ptr(tabs["bins"]), ptr(g),
                                 *(s // 4 for s in g.strides), y.shape[0], y.shape[1], hop, 128, 1e-5, chunk, ptr(out))
            assert rc == 0
            return out

        def forward(self, y, hop, n_frames):
            y = np.ascontiguousarray(y, f32)
            out = np.full((y.shape[0], 128, n_frames), np.nan, f32)
            assert lib.emu_mel_fwd(ptr(y), ptr(tabs["window"]), ptr(basis), ptr(tabs["lohi"]), y.shape[0], y.shape[1],
                                   hop, 128, 1e-5, ptr(out)) == 0
            return out

    return Emu()


@pytest.mark.parametrize("name", list(GG.CASES))
def test_backward_kernel_source_matches_reference_gradient(emu, name):
    z = np.load(GG.path(name))
    hop = int(z["hop"])
    ref = CF.mel_grad(z["y"], hop, z["cot"])
    floor = util.rms(z["grad"] - ref) / util.rms(ref)        # the fp32 reference's own error
    got = emu.backward(z["y"], hop, z["cot"], chunk=2 * hop)
    assert np.isfinite(got).all()
    e = util.rms(got - ref) / util.rms(ref)
    assert e <= RATIO * floor, (name, e, floor)
    assert util.rms(got - z["grad"]) / util.rms(ref) <= (RATIO + 1) * floor


@pytest.mark.parametrize("name", ["mel_grad_b1_f172_silence", "mel_grad_b1_hop256", "mel_grad_b1_short_constpad"])
def test_chunking_and_gradient_layout_do_not_change_a_bit(emu, name):
    """every sample is summed frame by frame in the same order whatever the chunk, and the transposed [B, F, n_mels]
    cotangent (extract's layout) is read in place"""
    z = np.load(GG.path(name))
    hop = int(z["hop"])
    a = emu.backward(z["y"], hop, z["cot"], chunk=2 * hop)
    b = emu.backward(z["y"], hop, z["cot"], chunk=8192)
    c = emu.backward(z["y"], hop, np.ascontiguousarray(z["cot"].transpose(0, 2, 1)).transpose(0, 2, 1), chunk=6 * hop)
    assert np.array_equal(a, b) and np.array_equal(a, c)


def test_forward_kernel_source_matches_reference_mel(emu):
    z = np.load(GG.path("mel_grad_b1_f172_silence"))
    got = emu.forward(z["y"], int(z["hop"]), z["mel"].shape[2])
    assert np.abs(got.astype(np.float64) - z["mel"]).max() < 2e-3


def test_backward_kernel_source_has_no_shared_memory_race(tmp_path):
    assert_race_free(tsan("tsan_mel_bwd.cpp", tmp_path))


def test_bin_filter_ranges_cover_every_weight():
    for args in ((44100, 2048, 128, 40, 16000), (44100, 2048, 80, 0, None)):
        basis = pm.mel_filterbank(*args)
        rng = pm._bin_filters(basis)
        assert rng.shape == (basis.shape[1], 2) and rng.dtype == np.int32
        for k in range(basis.shape[1]):
            col = basis[:, k]
            assert not col[:rng[k, 0]].any() and not col[rng[k, 1]:].any()
        assert (rng[:, 1] - rng[:, 0]).max() <= 3                # triangles: a bin lies under at most two filters


def test_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    ok = dict(audio=16, window=16, mel_basis=16, filter_lohi=16, bin_filter_range=16, B=1, n_samples=8192, n_fft=2048,
              win_size=2048, hop=512, n_mels=128, clip_val=1e-5, grad_mel=16, grad_stride_b=0, grad_stride_mel=16,
              grad_stride_frame=1, grad_audio=16, stream=0)
    call = lambda **kw: abi_call("b2d_mel_spectrogram_backward", dict(ok, **kw))
    assert call(audio=0) == -1 and call(bin_filter_range=0) == -1 and call(grad_mel=0) == -1             # B2D_ERR_NULL
    assert call(grad_audio=0) == -1
    assert call(B=0) == -2 and call(B=70000) == -2 and call(n_samples=0) == -2 and call(hop=4096) == -2    # B2D_ERR_SHAPE
    assert call(n_mels=129) == -2 and call(grad_stride_frame=-1) == -2 and call(grad_stride_mel=-128) == -2
    assert call(n_fft=1024, win_size=1024) == -4               # B2D_ERR_UNSUPPORTED: keyshift != 0
    assert b"mel_spectrogram_backward" in L.b2d_last_error()
