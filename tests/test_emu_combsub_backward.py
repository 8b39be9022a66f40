"""csrc/combsub_bwd.cu (the old-CombSub backward kernels) executed on the CPU (tests/emu/host_emu.h) against the
reference's autograd gradients (tests/golden/combsub_grad_*.npz) and the float64 closed form, race-checked under
ThreadSanitizer, plus the argument checks of its C ABI entry (no device touched).  The kernels run on hardware in
tests/test_gpu_combsub_backward.py.

The emulated kernels are fed the port's fp32 forward quantities (the reference's own comb, all-passed comb and harmonic
impulse responses), so the truth is the closed form at the reference's comb."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib
from oracle import torch_port as tp
from tests import util
from tests.golden import make_golden_combsub_grad as GG
from tests.test_oracle_combsub_grad import KEYS, error_model, load, reference_comb, split_grad

HERE = os.path.dirname(os.path.abspath(__file__))
P, SR = GG.P, GG.SR
f32 = np.float32

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("emu") / "libemu_combsub_bwd.so")
    cmd = ["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-Wno-unknown-pragmas",
           "-o", so, os.path.join(HERE, "emu", "emu_combsub_bwd.cpp")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    lib = ctypes.CDLL(so)
    fp = ctypes.POINTER(ctypes.c_float)
    lib.emu_combsub_bwd.argtypes = [fp, fp, fp, fp, ctypes.c_longlong, fp, fp, fp, fp, ctypes.c_ulonglong,
                                    ctypes.c_longlong, fp, fp, fp] + [ctypes.c_int] * 5 + [ctypes.c_double, fp, fp]

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


@needs_gxx
def test_backward_kernel_source_has_no_shared_memory_race(tmp_path):
    exe = str(tmp_path / "tsan_combsub_bwd")
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-pthread", "-Wno-unknown-pragmas", "-o", exe,
           os.path.join(HERE, "emu", "tsan_combsub_bwd.cpp")]
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
    f = L.b2d_combsub_synth_backward
    ws_need = L.b2d_combsub_synth_backward_workspace_bytes(1, 4, 512)
    assert ws_need == 4 * 512 * 4 and L.b2d_combsub_synth_backward_workspace_bytes(0, 4, 512) == 0
    ok = dict(f0=256, cg=256, ch=256, cn=256, stride=1024, noise=0, seed=0, off=0, fws=256, g=256, gh=0, gn=0, B=1,
              nF=4, block=512, Ma=256, Mh=512, Mn=256, sr=44100.0, out=256, ws=256, wsb=ws_need, stream=0)

    def call(**kw):
        a = dict(ok, **kw)
        return f(a["f0"], a["cg"], a["ch"], a["cn"], a["stride"], a["noise"], a["seed"], a["off"], a["fws"], a["g"],
                 a["gh"], a["gn"], a["B"], a["nF"], a["block"], a["Ma"], a["Mh"], a["Mn"], a["sr"], a["out"], a["ws"],
                 a["wsb"], a["stream"])

    assert call(fws=0) == -1 and call(out=0) == -1 and call(ws=0) == -1 and call(ch=0) == -1      # B2D_ERR_NULL
    assert call(B=0) == -2 and call(nF=0) == -2 and call(stride=500) == -2 and call(Mh=1) == -2    # B2D_ERR_SHAPE
    assert call(block=1024) == -4 and call(Mh=514, stride=1100) == -4 and call(B=65536) == -4     # UNSUPPORTED
    assert call(wsb=ws_need - 1) == -5                                                             # B2D_ERR_WORKSPACE
    assert call(ws=272) == -3 and call(fws=272) == -3 and call(noise=260) == -3                     # B2D_ERR_ALIGN
    assert b"combsub_synth_backward" in L.b2d_last_error()
