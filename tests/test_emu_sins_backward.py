"""csrc/sins_bwd.cu (the Sins backward kernels) executed on the CPU (tests/emu/host_emu.h) against the reference's
autograd gradients (tests/golden/sins_grad_*.npz), race-checked under ThreadSanitizer, plus the argument checks of
its C ABI entry (no device touched).  The kernels run on hardware in tests/test_gpu_sins_backward.py.

The emulated kernels are fed the port's fp32 forward quantities (sinusoids, impulse responses: the reference's own
values) and the phase scan's float64 frame phase."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from ddsp_svc_b200 import _lib
from oracle import torch_port as tp
from tests import sins_grad_closed_form as cfg
from tests import util
from tests.golden import make_golden_sins_grad as GG
from tests.test_oracle_sins_grad import KEYS, error_model, split_grad

HERE = os.path.dirname(os.path.abspath(__file__))
P, SR = GG.P, GG.SR
f32 = np.float32

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")


def frame_phase(f0):
    """b2d_phase_scan's fp64 unwrapped cycles at frame starts (phase_scan.cu), [B, nF]"""
    f = np.asarray(f0, np.float64).reshape(f0.shape[0], -1)
    fn = np.concatenate([f[:, 1:], f[:, -1:]], axis=1)
    adv = (P * f + (fn - f) * 0.5 * (P - 1)) / SR
    return np.ascontiguousarray(np.concatenate([np.zeros((f.shape[0], 1)), np.cumsum(adv, axis=1)[:, :-1]], axis=1))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("emu") / "libemu_sins_bwd.so")
    cmd = ["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-Wno-unknown-pragmas",
           "-o", so, os.path.join(HERE, "emu", "emu_sins_bwd.cpp")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    lib = ctypes.CDLL(so)
    fp, dp = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_double)
    lib.emu_sins_bwd.argtypes = [fp, dp, fp, fp, fp, ctypes.c_longlong, fp, fp, fp, fp, ctypes.c_ulonglong,
                                 ctypes.c_longlong, fp, fp, fp] + [ctypes.c_int] * 5 + [ctypes.c_double, fp, fp]

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


@needs_gxx
def test_backward_kernel_source_has_no_shared_memory_race(tmp_path):
    exe = str(tmp_path / "tsan_sins_bwd")
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-pthread", "-Wno-unknown-pragmas", "-o", exe,
           os.path.join(HERE, "emu", "tsan_sins_bwd.cpp")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0 and "tsan" in proc.stderr.lower():
        pytest.skip("ThreadSanitizer runtime not available: " + proc.stderr.strip().splitlines()[-1])
    assert proc.returncode == 0, proc.stderr
    res = subprocess.run([exe], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66"))
    assert "ThreadSanitizer" not in res.stderr, res.stderr[-4000:]
    assert res.returncode == 0 and "done" in res.stdout


def test_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    f = L.b2d_sins_synth_backward
    ws_need = L.b2d_sins_synth_backward_workspace_bytes(1, 4, 512)
    assert ws_need == 2 * 4 * 512 * 4 and L.b2d_sins_synth_backward_workspace_bytes(0, 4, 512) == 0
    ok = dict(f0=256, fph=256, ca=256, cg=256, cn=256, stride=640, noise=0, seed=0, off=0, fws=256, has=1, g=256, gh=0,
              gn=0, B=1, nF=4, block=512, H=128, Ma=256, Mn=256, sr=44100.0, out=256, ws=256, wsb=ws_need, stream=0)

    def call(**kw):
        a = dict(ok, **kw)
        return f(a["f0"], a["fph"], a["ca"], a["cg"], a["cn"], a["stride"], a["noise"], a["seed"], a["off"], a["fws"],
                 a["has"], a["g"], a["gh"], a["gn"], a["B"], a["nF"], a["block"], a["H"], a["Ma"], a["Mn"], a["sr"],
                 a["out"], a["ws"], a["wsb"], a["stream"])

    assert call(fws=0) == -1 and call(out=0) == -1 and call(ws=0) == -1 and call(cg=0) == -1      # B2D_ERR_NULL
    assert call(B=0) == -2 and call(nF=0) == -2 and call(stride=200) == -2 and call(Ma=1) == -2    # B2D_ERR_SHAPE
    assert call(block=1024) == -4 and call(Ma=258, stride=700) == -4 and call(H=513, stride=1100) == -4   # UNSUPPORTED
    assert call(wsb=ws_need - 1) == -5                                                             # B2D_ERR_WORKSPACE
    assert call(ws=272) == -3 and call(fws=272) == -3 and call(noise=260) == -3                     # B2D_ERR_ALIGN
    assert b"sins_synth_backward" in L.b2d_last_error()
