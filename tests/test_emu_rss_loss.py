"""csrc/rss_loss.cu's kernel sources executed on the CPU (tests/emu/host_emu.h) against the reference's autograd goldens
(tests/golden/rss_*.npz) and the float64 restatement, race-checked under ThreadSanitizer, plus the argument checks of
the C ABI entries (no device touched).  The kernels themselves run on hardware in tests/test_gpu_rss_loss.py."""
import ctypes

import numpy as np
import pytest

from ddsp_svc_b200 import _lib
from ddsp_svc_b200 import loss as pl
from tests import rss_loss_closed_form as CF
from tests import report, util
from tests.emu_harness import abi_call, assert_race_free, shared, tsan
from tests.golden import make_golden_rss_loss as GR

f32 = np.float32
# error model (see tests/test_gpu_rss_loss.py): against float64 the loss (relative) and the gradient (relative RMS) stay
# within RATIO times the fp32 reference's own error on the same case (the loss floor: at least one fp32 ulp)
RATIO = 3.0


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_rss_loss.cpp", tmp_path_factory)
    _lib.build()
    vp, ci = ctypes.c_void_p, ctypes.c_int
    ptr = lambda a: a.ctypes.data_as(vp)

    class Emu:
        def run(self, x_pred, x_true, n_ffts):
            """-> loss, norms [n_scale, B, 2], dL/dx_pred"""
            xp = np.ascontiguousarray(x_pred, f32)
            xt = np.ascontiguousarray(np.asarray(x_true).astype(f32))
            B, T = xp.shape
            tabs = [pl.table_host(n) for n in n_ffts]
            tp = (vp * len(n_ffts))(*[t.ctypes.data for t in tabs])
            ns = (ci * len(n_ffts))(*n_ffts)
            part = np.zeros(lib.emu_rss_workspace_doubles(B, T, len(n_ffts), ns))
            norms = np.zeros((len(n_ffts), B, 2))
            loss = np.zeros(1, f32)
            assert lib.emu_rss_forward(ptr(xp), ptr(xt), B, T, len(n_ffts), ns, tp, 1.0, 1e-7, ptr(part), ptr(norms),
                                       ptr(loss)) == 0
            gl = np.ones(1, f32)
            dx = np.full((B, T), np.nan, f32)
            assert lib.emu_rss_backward(ptr(xp), ptr(xt), B, T, len(n_ffts), ns, tp, 1.0, 1e-7, ptr(norms), ptr(gl),
                                        ptr(dx)) == 0
            return float(loss[0]), norms, dx

        def spectra(self, x_pred, x_true, n):
            """-> S_p, S_t [B, F, K] as the kernels compute them"""
            xp = np.ascontiguousarray(x_pred, f32)
            xt = np.ascontiguousarray(np.asarray(x_true).astype(f32))
            B, T = xp.shape
            F, K = 1 + (T - n) // n, n // 2 + 1
            sp, st = np.full((B, F, K), np.nan, f32), np.full((B, F, K), np.nan, f32)
            tab = pl.table_host(n)
            assert lib.emu_rss_spectra(ptr(xp), ptr(xt), B, T, n, ptr(tab), 1e-7, ptr(sp), ptr(st)) == 0
            return sp, st

    return Emu()


@pytest.mark.parametrize("name", list(GR.CASES))
def test_kernel_source_matches_reference_within_error_model(emu, name):
    z = np.load(GR.path(name))
    n_ffts = [int(v) for v in z["n_ffts"]]
    xt = z["x_true"].astype(f32)
    ref_loss, ref_grad, ref_norms = CF.loss_and_grad(z["x_pred"], xt, n_ffts)
    floor_l = max(abs(float(z["loss"]) - ref_loss), float(np.spacing(f32(ref_loss)))) / ref_loss
    floor_g = util.rms(z["grad"] - ref_grad) / util.rms(ref_grad)
    loss, norms, grad = emu.run(z["x_pred"], z["x_true"], n_ffts)
    assert np.isfinite(grad).all()
    assert abs(loss - ref_loss) / ref_loss <= RATIO * floor_l, (loss, ref_loss, floor_l)
    assert util.rms(grad - ref_grad) / util.rms(ref_grad) <= RATIO * floor_g
    assert util.rms(grad - z["grad"]) / util.rms(ref_grad) <= (RATIO + 1) * floor_g
    assert np.allclose(norms, ref_norms, rtol=1e-4, atol=0)


def _spectra64(x, n, eps=1e-7):
    B, T = x.shape
    F = 1 + (T - n) // n
    w = CF.hann(n)
    return np.abs(np.fft.rfft(np.asarray(x, np.float64)[:, :F * n].reshape(B, F, n) * w, axis=-1)) / np.sqrt(
        np.sum(w * w)) + eps


@pytest.mark.parametrize("name", list(GR.CASES))
def test_kernel_sign_disagreements_with_float64_are_counted(emu, name):
    """the bins where the kernels' sign(log S_t - log S_p) differs from float64's: the 1 / S_p term of those bins is
    what the gradient error model has to absorb.  Counted for the kernel source and for the fp32 oracle, recorded, and
    held to the same order (each is a rounding coin-toss in bins where the two logs agree to ~1e-6)."""
    import torch
    from oracle import loss as ol
    z = np.load(GR.path(name))
    xp, xt = z["x_pred"], z["x_true"].astype(f32)
    kern = orac = bins = 0
    for n in (int(v) for v in z["n_ffts"]):
        sp, st = emu.spectra(xp, xt, n)
        s64 = np.sign(np.log(_spectra64(xt, n)) - np.log(_spectra64(xp, n)))
        kern += int((np.sign(np.log(st) - np.log(sp)) != s64).sum())
        o32 = (torch.log(ol.spectrogram(torch.from_numpy(xt), n, n) + 1e-7) -
               torch.log(ol.spectrogram(torch.from_numpy(xp), n, n) + 1e-7)).sign().numpy().transpose(0, 2, 1)
        orac += int((o32 != s64).sum())
        bins += s64.size
    report.record("rss_loss_emu/sign_flips_" + name, kernel=kern, oracle_fp32=orac, bins=bins)
    assert kern <= max(4, 4 * orac), (kern, orac, bins)


def test_equal_row_is_exactly_zero_and_rows_do_not_depend_on_the_batch(emu):
    """every row's norms and gradient direction come from its own frames only, whatever the batch around it: a row
    alone gives bit-identical norms, and B times its in-batch gradient up to the final fp32 scaling"""
    z = np.load(GR.path("rss_equal_row"))
    n_ffts = [int(v) for v in z["n_ffts"]]
    loss, norms, grad = emu.run(z["x_pred"], z["x_true"], n_ffts)
    assert not np.any(grad[1]) and np.all(norms[:, 1, 0] == 0)
    alone_loss, alone_norms, _ = emu.run(z["x_pred"][1:2], z["x_true"][1:2], n_ffts)
    assert alone_loss == 0.0
    for r in (0, 2):
        _, nr, _ = emu.run(z["x_pred"][r:r + 1], z["x_true"][r:r + 1], n_ffts)
        assert np.array_equal(nr[:, 0], norms[:, r])


def test_samples_past_the_last_frame_get_zero(emu):
    z = np.load(GR.path("rss_ragged_t"))
    n_ffts = [int(v) for v in z["n_ffts"]]
    T = z["x_pred"].shape[1]
    end = max((T // n) * n for n in n_ffts)
    _, _, grad = emu.run(z["x_pred"], z["x_true"], n_ffts)
    assert not np.any(grad[:, end:]) and np.isfinite(grad).all()


def test_scale_order_changes_only_the_summation(emu):
    z = np.load(GR.path("rss_ragged_t"))
    n_ffts = [int(v) for v in z["n_ffts"]]
    l1, n1, g1 = emu.run(z["x_pred"], z["x_true"], n_ffts)
    l2, n2, g2 = emu.run(z["x_pred"], z["x_true"], n_ffts[::-1])
    assert np.array_equal(n1, n2[::-1])
    assert util.rms(g1 - g2) <= 1e-6 * util.rms(g1)


def test_kernel_source_has_no_shared_memory_race(tmp_path):
    assert_race_free(tsan("tsan_rss_loss.cpp", tmp_path))


def test_table_layout_and_bluestein_sizes():
    _lib.build()
    L = _lib.lib()
    for n in (256, 512, 513, 1024, 1025, 2047):
        M = pl.bluestein_size(n)
        assert M >= 2 * n - 1 and (M == 1024 or M // 2 < 2 * n - 1)
        t = pl.table_host(n)
        assert t.size == L.b2d_rss_table_floats(n)
        co = 4 + ((n + 3) & ~3)
        chirp = t[co:co + 2 * n].view(np.complex64)
        m = np.arange(n)
        assert np.allclose(chirp, np.exp(1j * np.pi * (m * m % (2 * n)) / n), atol=1e-7)
    assert L.b2d_rss_table_floats(255) == 0 and L.b2d_rss_table_floats(2048) == 0
    assert L.b2d_rss_frames(5003, 1031) == 4 and L.b2d_rss_frames(100, 256) == 0


def test_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    ns = (ctypes.c_int * 2)(512, 1031)
    tabs = (ctypes.c_void_p * 2)(256, 512)
    bad_n = (ctypes.c_int * 1)(2048)
    common = dict(x_pred=16, x_true=16, B=2, n_samples=8192, n_scale=2, n_ffts=ns, tables=tabs, alpha=1.0, eps=1e-7,
                  norms=16, stream=0)
    ok_fwd = dict(common, workspace=16, workspace_bytes=1 << 20, loss=16)
    ok_bwd = dict(common, grad_loss=16, grad_pred=16)
    fwd = lambda **kw: abi_call("b2d_rss_loss_forward", dict(ok_fwd, **kw))
    bwd = lambda **kw: abi_call("b2d_rss_loss_backward", dict(ok_bwd, **kw))
    for f, scalar in ((fwd, "loss"), (bwd, "grad_loss")):       # the loss, or the cotangent of the loss
        assert f(x_pred=0) == -1 and f(x_true=0) == -1 and f(norms=0) == -1 and f(**{scalar: 0}) == -1   # B2D_ERR_NULL
        assert f(tables=(ctypes.c_void_p * 2)(256, 0)) == -1
        assert f(x_pred=18) == -3 and f(norms=20) == -3 and f(tables=(ctypes.c_void_p * 2)(256, 260)) == -3   # ALIGN
        assert f(B=0) == -2 and f(B=70000) == -2 and f(n_samples=1000) == -2 and f(n_scale=65) == -2   # B2D_ERR_SHAPE
        assert f(n_ffts=bad_n, n_scale=1) == -4 and f(n_ffts=(ctypes.c_int * 1)(255), n_scale=1) == -4  # UNSUPPORTED
    assert fwd(workspace_bytes=8) == -5                                                        # B2D_ERR_WORKSPACE
    assert b"rss_loss" in L.b2d_last_error()
    assert L.b2d_rss_loss_workspace_bytes(2, 8192, 2, ns) == 8 * 3 * 2 * (16 + 7)
