"""csrc/reflow.cu's kernel source (start, layer epilogue, ODE update, finish of the rectified-flow sampler) executed on
the CPU (tests/emu/host_emu.h) against float64 restatements, race-checked under ThreadSanitizer, plus the argument
checks of the new C ABI entries (no device touched).  The kernels run on hardware in tests/test_gpu_reflow.py."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("emu") / "libemu_reflow.so")
    cmd = ["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-Wno-unknown-pragmas",
           "-o", so, os.path.join(HERE, "emu", "emu_reflow.cpp")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    lib = ctypes.CDLL(so)
    p, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    lib.emu_rf_start.argtypes = [p, p, f, f, f, f, i, i, i, p, p, p]
    lib.emu_rf_layer_input.argtypes = [p, p, p, i, p, i, p, i, i, i, i, p, p]
    lib.emu_rf_ode.argtypes = [p, p, p, p, i, f, i, i, p, p]
    lib.emu_rf_finish.argtypes = [p, f, f, i, p]
    return lib


def f32(a):
    return np.ascontiguousarray(np.asarray(a, np.float32))


def ptr(a):
    return None if a is None else a.ctypes.data


def out_buffers(shape, split):
    hi = np.full(shape, np.nan, np.float32)
    return hi, (np.full(shape, np.nan, np.float32) if split else None)


def check_operand(hi, lo, want, rel=1e-6):
    """hi (+ lo) against the float64 value; split halves must be TF32-exact (low 13 mantissa bits zero)"""
    got = hi.astype(np.float64) + (0 if lo is None else lo.astype(np.float64))
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= rel * scale, np.abs(got - want).max() / scale
    if lo is not None:
        for part in (hi, lo):
            assert not (part.view(np.uint32) & 0x1FFF).any()
        assert np.abs(lo).max() <= 2.0 ** -10 * np.abs(hi).max()


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("with_gt", [False, True])
def test_start_kernel(emu, split, with_gt):
    rng = np.random.default_rng(1 + split + 2 * with_gt)
    B, T, M = 2, 11, 12
    noise, gt = f32(rng.standard_normal((B, 1, M, T))), f32(rng.standard_normal((B, T, M)) * 3 - 5)
    x = np.full((B, T, M), np.nan, np.float32)
    hi, lo = out_buffers((B, T, M), split)
    ts = 0.7 if with_gt else 0.0
    emu.emu_rf_start(ptr(noise), ptr(gt) if with_gt else None, ts, 1.0 - ts, -12.0, 14.0, B, T, M, ptr(x), ptr(hi), ptr(lo))
    want = noise[:, 0].transpose(0, 2, 1).astype(np.float64)
    if with_gt:
        want = 0.7 * ((gt.astype(np.float64) + 12) / 14 * 2 - 1) + 0.3 * want
    assert np.abs(x - want).max() <= 1e-6 * np.abs(want).max()
    check_operand(hi, lo, want)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("residual", [0, 1])
@pytest.mark.parametrize("cond_mode", ["per_utterance", "shared_step", "last_layer"])
def test_layer_input_kernel(emu, split, residual, cond_mode):
    rng = np.random.default_rng(10 * residual + split + 3 * len(cond_mode))
    B, T, D, L, layer = 2, 9, 64, 3, 1
    LD = L * D
    g, bias, h0 = (f32(rng.standard_normal(s)) for s in ((B, T, D), (D,), (B, T, D)))
    steps = f32(rng.standard_normal((B, LD)))
    cond = f32(rng.standard_normal((B, T, LD)))
    h = h0.copy()
    hi, lo = out_buffers((B, T, D), split)
    stride = {"per_utterance": LD, "shared_step": 0, "last_layer": 0}[cond_mode]
    sp = None if cond_mode == "last_layer" else steps.ctypes.data + 4 * layer * D
    cp = None if cond_mode == "last_layer" else cond.ctypes.data + 4 * layer * D
    assert emu.emu_rf_layer_input(ptr(g), ptr(bias), ptr(h), residual, sp, stride, cp, LD, B, T, D, ptr(hi), ptr(lo)) == 0
    pre = g.astype(np.float64) + bias
    want_h = pre + h0 if residual else torch.nn.functional.gelu(torch.from_numpy(pre)).numpy()
    assert np.abs(h - want_h).max() <= 1e-6 * np.abs(want_h).max()
    want_u = want_h.copy()
    if cond_mode != "last_layer":
        srow = steps[:, None, layer * D:(layer + 1) * D] if stride else steps[0][None, None, layer * D:(layer + 1) * D]
        want_u = want_u + srow + cond[:, :, layer * D:(layer + 1) * D]
    check_operand(hi, lo, want_u)


@pytest.mark.parametrize("split", [False, True])
def test_ode_kernel_euler_and_rk4(emu, split):
    rng = np.random.default_rng(5 + split)
    N, M, dt = 23, 12, 0.05
    bias = f32(rng.standard_normal(M))
    x0 = f32(rng.standard_normal((N, M)))
    # Euler
    x, G = x0.copy(), f32(rng.standard_normal((N, M)))
    hi, lo = out_buffers((N, M), split)
    emu.emu_rf_ode(ptr(G), ptr(bias), ptr(x), None, -1, dt, N, M, ptr(hi), ptr(lo))
    want = x0.astype(np.float64) + (G.astype(np.float64) + bias) * np.float32(dt)
    assert np.abs(x - want).max() <= 1e-6 * np.abs(want).max()
    check_operand(hi, lo, want)
    # RK4: four stages with independent "velocities"
    x, acc = x0.copy(), np.full((N, M), np.nan, np.float32)
    ks = [f32(rng.standard_normal((N, M))) for _ in range(4)]
    coef = [0.5, 0.5, 1.0]
    for s, Gs in enumerate(ks):
        hi, lo = out_buffers((N, M), split)
        emu.emu_rf_ode(ptr(Gs), ptr(bias), ptr(x), ptr(acc), s, dt, N, M, ptr(hi), ptr(lo))
        k = [kk.astype(np.float64) + bias for kk in ks]
        if s < 3:
            assert np.array_equal(x, x0)
            check_operand(hi, lo, x0 + coef[s] * k[s] * np.float32(dt))
    want = x0 + (k[0] + 2 * k[1] + 2 * k[2] + k[3]) * np.float32(dt) / 6
    assert np.abs(x - want).max() <= 2e-6 * np.abs(want).max()
    check_operand(hi, lo, want, rel=2e-6)


def test_finish_kernel(emu):
    x = f32(np.random.default_rng(3).standard_normal(77))
    out = np.full(77, np.nan, np.float32)
    emu.emu_rf_finish(ptr(x), -12.0, 14.0, 77, ptr(out))
    want = (x.astype(np.float64) + 1) / 2 * 14 - 12
    assert np.abs(out - want).max() <= 1e-6 * np.abs(want).max()


@needs_gxx
def test_reflow_kernel_source_has_no_race(tmp_path):
    exe = str(tmp_path / "tsan_reflow")
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-pthread", "-Wno-unknown-pragmas", "-o", exe,
           os.path.join(HERE, "emu", "tsan_reflow.cpp")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0 and "tsan" in proc.stderr.lower():
        pytest.skip("ThreadSanitizer runtime not available: " + proc.stderr.strip().splitlines()[-1])
    assert proc.returncode == 0, proc.stderr
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66"))
    assert "ThreadSanitizer" not in res.stderr, res.stderr[-4000:]
    assert res.returncode == 0 and "done" in res.stdout


def test_reflow_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    p = 16                                                     # a non-null, 16-byte aligned address
    assert L.b2d_rf_start(0, 0, 0.0, 1.0, -12.0, 14.0, 1, 8, 128, 0, p, 0, 0) == -1
    assert L.b2d_rf_start(p, 0, 0.0, 1.0, -12.0, 14.0, 1, 8, 128, 0, 0, 0, 0) == -1
    assert L.b2d_rf_start(p, 0, 0.0, 1.0, -12.0, 14.0, 1, 0, 128, 0, p, 0, 0) == -2
    li = lambda **kw: L.b2d_rf_layer_input(*[{**dict(g=p, b=p, h=p, r=0, s=p, ss=0, c=p, cs=1536, B=1, T=8, D=512, hi=p, lo=0,
                                                     st=0), **kw}[k]
                                             for k in ("g", "b", "h", "r", "s", "ss", "c", "cs", "B", "T", "D", "hi", "lo", "st")])
    assert li(g=0) == -1 and li(hi=0) == -1 and li(c=0) == -1 and li(s=0) == -1       # step and cond come together
    assert li(B=0) == -2 and li(ss=100) == -2 and li(cs=256) == -2
    assert li(D=510, cs=1530) == -3 and li(g=p + 4) == -3 and li(s=p + 4) == -3 and li(cs=1538) == -3
    assert b"rf_layer_input" in L.b2d_last_error()
    ode = lambda **kw: L.b2d_rf_ode_update(*[{**dict(g=p, b=p, x=p, a=p, s=0, dt=0.1, n=8, M=128, hi=p, lo=0, st=0), **kw}[k]
                                             for k in ("g", "b", "x", "a", "s", "dt", "n", "M", "hi", "lo", "st")])
    assert ode(a=0) == -1 and ode(x=0) == -1 and ode(n=0) == -2 and ode(s=4) == -4 and ode(s=-2) == -4
    assert L.b2d_rf_finish(0, -12.0, 14.0, 8, p, 0) == -1 and L.b2d_rf_finish(p, -12.0, 14.0, 0, p, 0) == -2
