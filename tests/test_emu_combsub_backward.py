"""csrc/combsub_bwd.cu (the old-CombSub backward kernels) executed on the CPU (tests/emu/host_emu.h) against the
reference's autograd gradients (tests/golden/combsub_grad_*.npz) and the float64 closed form, race-checked under
ThreadSanitizer, plus the argument checks of its C ABI entry (no device touched).  The kernels run on hardware in
tests/test_gpu_combsub_backward.py.

The emulated kernels are fed the port's fp32 forward quantities (the reference's own comb, all-passed comb and harmonic
impulse responses), so the truth is the closed form at the reference's comb."""
import ctypes

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib
from oracle import torch_port as tp
from tests import util
from tests.emu_harness import abi_call, assert_race_free, shared, tsan
from tests.golden import make_golden_combsub_grad as GG
from tests.test_oracle_combsub_grad import KEYS, error_model, load, reference_comb, split_grad

P, SR = GG.P, GG.SR
f32 = np.float32


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_combsub_bwd.cpp", tmp_path_factory)
    fp = ctypes.POINTER(ctypes.c_float)

    def run(inp, noise="explicit", seed=0, utt_off=0, rows=None):
        c = inp["case"]
        Ma, Mh, Mn = c["Ma"], c["Mh"], c["Mn"]
        sel = slice(None) if rows is None else rows
        with torch.no_grad():
            fwd = tp.combsub_forward(inp["f0"], inp["ctrls"], SR, P, noise=inp["noise"], infer=False)
        arr = lambda t: None if t is None else np.ascontiguousarray(np.asarray(t.numpy())[sel], f32)
        f0 = arr(inp["f0"])
        dense = arr(inp["dense"])
        comb, allp, ir_h, nz = arr(fwd["comb"]), arr(fwd["allpassed"]), arr(fwd["ir_harmonic"]), arr(inp["noise"])
        g, gh, gn = arr(inp["cot"]), arr(inp["cot_h"]), arr(inp["cot_n"])
        B, nF = f0.shape[0], f0.shape[1]
        da = np.full((B, nF * P), np.nan, f32)
        out = np.full((B, nF, Ma + Mh + Mn), np.nan, f32)
        ptr = lambda a, off=0: None if a is None else ctypes.cast(a.ctypes.data + a.itemsize * off, fp)
        rc = lib.emu_combsub_bwd(ptr(f0), ptr(dense), ptr(dense, Ma), ptr(dense, Ma + Mh), Ma + Mh + Mn, ptr(comb),
                                 ptr(allp), ptr(ir_h), ptr(nz) if noise == "explicit" else None, seed, utt_off, ptr(g),
                                 ptr(gh), ptr(gn), B, nF, Ma, Mh, Mn, float(SR), ptr(da), ptr(out))
        assert rc == 0
        return out

    return run


@pytest.mark.parametrize("name", list(GG.CASES))
def test_backward_kernel_source_matches_reference_gradient(emu, name):
    inp, gold = load(name)
    truth, bound, _ = error_model(name, inp, gold["grad"], reference_comb(inp))
    got = split_grad(name, emu(inp))
    for k in KEYS:
        assert np.isfinite(got[k]).all()
        e = util.rms(got[k] - truth[k]) / util.rms(truth[k])
        assert e <= bound[k], (name, k, e, bound[k])


def test_in_kernel_noise_rows_are_shard_invariant(emu):
    inp, _ = load("combsub_grad_b2_f6_parts")
    full = emu(inp, noise="kernel", seed=3)
    part = emu(inp, noise="kernel", seed=3, utt_off=1, rows=slice(1, 2))
    assert np.isfinite(full).all() and np.array_equal(full[1:], part)
    assert not np.array_equal(full, emu(inp, noise="kernel", seed=4))


def test_backward_kernel_source_has_no_shared_memory_race(tmp_path):
    assert_race_free(tsan("tsan_combsub_bwd.cpp", tmp_path))


def test_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    ws_need = L.b2d_combsub_synth_backward_workspace_bytes(1, 4, 512)
    assert ws_need == 4 * 512 * 4 and L.b2d_combsub_synth_backward_workspace_bytes(0, 4, 512) == 0
    ok = dict(f0_frames=256, c_group_delay=256, c_harmonic=256, c_noise=256, ctrl_stride=1024, noise_in=0, seed=0,
              utterance_offset=0, forward_workspace=256, grad_signal=256, grad_harmonic=0, grad_noise=0, B=1, n_frames=4,
              block=512, n_mag_allpass=256, n_mag_harmonic=512, n_mag_noise=256, sampling_rate=44100.0, grad_ctrl=256,
              workspace=256, workspace_bytes=ws_need, stream=0)
    call = lambda **kw: abi_call("b2d_combsub_synth_backward", dict(ok, **kw))
    assert call(forward_workspace=0) == -1 and call(grad_ctrl=0) == -1 and call(workspace=0) == -1     # B2D_ERR_NULL
    assert call(c_harmonic=0) == -1
    assert call(B=0) == -2 and call(n_frames=0) == -2 and call(ctrl_stride=500) == -2                  # B2D_ERR_SHAPE
    assert call(n_mag_harmonic=1) == -2
    assert call(block=1024) == -4 and call(n_mag_harmonic=514, ctrl_stride=1100) == -4                 # UNSUPPORTED
    assert call(B=65536) == -4
    assert call(workspace_bytes=ws_need - 1) == -5                                                     # B2D_ERR_WORKSPACE
    assert call(workspace=272) == -3 and call(forward_workspace=272) == -3 and call(noise_in=260) == -3  # B2D_ERR_ALIGN
    assert b"combsub_synth_backward" in L.b2d_last_error()
