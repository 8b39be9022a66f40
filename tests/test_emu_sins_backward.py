"""csrc/sins_bwd.cu (the Sins backward kernels) executed on the CPU (tests/emu/host_emu.h) against the reference's
autograd gradients (tests/golden/sins_grad_*.npz), race-checked under ThreadSanitizer, plus the argument checks of
its C ABI entry (no device touched).  The kernels run on hardware in tests/test_gpu_sins_backward.py.

The emulated kernels are fed the port's fp32 forward quantities (sinusoids, impulse responses: the reference's own
values) and the phase scan's float64 frame phase."""
import ctypes

import numpy as np
import pytest

from ddsp_svc_b200 import _lib
from oracle import torch_port as tp
from tests import sins_grad_closed_form as cfg
from tests import util
from tests.emu_harness import abi_call, assert_race_free, shared, tsan
from tests.golden import make_golden_sins_grad as GG
from tests.test_oracle_sins_grad import KEYS, error_model, split_grad

P, SR = GG.P, GG.SR
f32 = np.float32


def frame_phase(f0):
    """b2d_phase_scan's fp64 unwrapped cycles at frame starts (phase_scan.cu), [B, nF]"""
    f = np.asarray(f0, np.float64).reshape(f0.shape[0], -1)
    fn = np.concatenate([f[:, 1:], f[:, -1:]], axis=1)
    adv = (P * f + (fn - f) * 0.5 * (P - 1)) / SR
    return np.ascontiguousarray(np.concatenate([np.zeros((f.shape[0], 1)), np.cumsum(adv, axis=1)[:, :-1]], axis=1))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_sins_bwd.cpp", tmp_path_factory)
    fp, dp = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)

    def run(name, inp, noise="explicit", seed=0, utt_off=0, rows=None):
        c = GG.CASES[name]
        H, Ma, Mn = c["H"], c["Ma"], c["Mn"]
        sel = slice(None) if rows is None else rows
        f0 = np.ascontiguousarray(inp["f0"].numpy()[sel], f32)
        fwd = tp.sins_forward(inp["f0"], inp["ctrls"], SR, P, noise=inp["noise"], infer=False)
        arr = lambda t: np.ascontiguousarray(np.asarray(t.detach().numpy() if hasattr(t, "detach") else t)[sel], f32)
        # the sinusoids the GPU forward produces: the bank at the kernels' phase
        sinus = cfg.sinusoids(inp["f0"].numpy(), inp["ctrls"]["amplitudes"].numpy(),
                              cfg.kernel_phase(inp["f0"].numpy(), SR, P), SR, P, reference_rounding=False)
        dense, sinus = arr(inp["dense"]), arr(sinus)
        ir_ap, ir_n, nz = arr(fwd["ir_allpass"]), arr(fwd["ir_noise"]), arr(inp["noise"])
        g = arr(inp["cot"])
        gh = None if inp["cot_h"] is None else arr(inp["cot_h"])
        gn = None if inp["cot_n"] is None else arr(inp["cot_n"])
        fph = frame_phase(f0)
        B, nF = f0.shape[0], f0.shape[1]
        dx = np.full((B, nF * P), np.nan, f32)
        out = np.full((B, nF, H + Ma + Mn), np.nan, f32)
        ptr = lambda a, off=0: None if a is None else ctypes.cast(a.ctypes.data + a.itemsize * off,
                                                                    dp if a.dtype == np.float64 else fp)
        rc = lib.emu_sins_bwd(ptr(f0), ptr(fph), ptr(dense), ptr(dense, H), ptr(dense, H + Ma), H + Ma + Mn, ptr(sinus),
                              ptr(ir_ap), ptr(ir_n), ptr(nz) if noise == "explicit" else None, seed, utt_off, ptr(g),
                              ptr(gh), ptr(gn), B, nF, H, Ma, Mn, float(SR), ptr(dx), ptr(out))
        assert rc == 0
        return out

    return run


# relative RMS per control against float64 at the kernels' phase, as a multiple of the fp32 reference's own error
# against float64 at its phase (tests/test_oracle_sins_grad.error_model): the kernels use fp32 direct-form sums where
# the reference uses fp32 FFTs, and an exactly reduced sine where it rounds 2 pi h x to fp32
RATIO = 3.0
# ... but not below the random-rounding floor of one fp32 sum of 2P products (every dh tap sums 1024 of them; the
# reference's FFTs of very short filters sum far fewer)
FLOOR = 2.0 ** -24 * np.sqrt(2 * P)


@pytest.mark.parametrize("name", list(GG.CASES))
def test_backward_kernel_source_matches_reference_gradient(emu, name):
    inp = GG.build_inputs(name)
    truth, ref_err = error_model(inp, np.load(GG.path(name))["grad"], name)
    got = split_grad(name, emu(name, inp))
    for k in KEYS:
        assert np.isfinite(got[k]).all()
        e = util.rms(got[k] - truth[k]) / util.rms(truth[k])
        assert e <= max(RATIO * ref_err[k], FLOOR), (name, k, e, ref_err[k])


def test_in_kernel_noise_rows_are_shard_invariant(emu):
    name = "sins_grad_b2_f24_h128"
    inp = GG.build_inputs(name)
    full = emu(name, inp, noise="kernel", seed=3)
    part = emu(name, inp, noise="kernel", seed=3, utt_off=1, rows=slice(1, 2))
    assert np.isfinite(full).all() and np.array_equal(full[1:], part)
    assert not np.array_equal(full, emu(name, inp, noise="kernel", seed=4))


def test_backward_kernel_source_has_no_shared_memory_race(tmp_path):
    assert_race_free(tsan("tsan_sins_bwd.cpp", tmp_path))


def test_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    ws_need = L.b2d_sins_synth_backward_workspace_bytes(1, 4, 512)
    assert ws_need == 2 * 4 * 512 * 4 and L.b2d_sins_synth_backward_workspace_bytes(0, 4, 512) == 0
    ok = dict(f0_frames=256, frame_phase=256, c_amp=256, c_group_delay=256, c_noise=256, ctrl_stride=640, noise_in=0,
              seed=0, utterance_offset=0, forward_workspace=256, forward_has_sinusoids=1, grad_signal=256,
              grad_harmonic=0, grad_noise=0, B=1, n_frames=4, block=512, n_harmonics=128, n_mag_allpass=256,
              n_mag_noise=256, sampling_rate=44100.0, grad_ctrl=256, workspace=256, workspace_bytes=ws_need, stream=0)
    call = lambda **kw: abi_call("b2d_sins_synth_backward", dict(ok, **kw))
    assert call(forward_workspace=0) == -1 and call(grad_ctrl=0) == -1 and call(workspace=0) == -1     # B2D_ERR_NULL
    assert call(c_group_delay=0) == -1
    assert call(B=0) == -2 and call(n_frames=0) == -2 and call(ctrl_stride=200) == -2                  # B2D_ERR_SHAPE
    assert call(n_mag_allpass=1) == -2
    assert call(block=1024) == -4 and call(n_mag_allpass=258, ctrl_stride=700) == -4                   # UNSUPPORTED
    assert call(n_harmonics=513, ctrl_stride=1100) == -4
    assert call(workspace_bytes=ws_need - 1) == -5                                                     # B2D_ERR_WORKSPACE
    assert call(workspace=272) == -3 and call(forward_workspace=272) == -3 and call(noise_in=260) == -3  # B2D_ERR_ALIGN
    assert b"sins_synth_backward" in L.b2d_last_error()
