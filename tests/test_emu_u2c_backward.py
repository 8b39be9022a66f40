"""csrc/unit2control_bwd.cu's GLU -> depthwise conv -> SiLU backward kernel source executed on the CPU
(tests/emu/host_emu.h) against autograd of the same op in float64, race-checked under ThreadSanitizer, plus the argument
checks of the new C ABI entries (no device touched).  The kernels run on hardware in
tests/test_gpu_unit2control_backward.py."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import _lib
from tests import util

HERE = os.path.dirname(os.path.abspath(__file__))
needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")


def glu_dwconv_silu_reference(h, w, bias, gout):
    """float64 autograd of GLU -> depthwise Conv1d(k = 31, padding 15) -> SiLU on token-major h [B, T, 2 Ci]
    -> (gh [B, T, 2 Ci], dwb [Ci, 32]: 31 tap gradients, then the bias gradient)"""
    h, w, bias = (t.double().requires_grad_(True) for t in (h, w, bias))
    Ci = w.shape[0]
    u = F.glu(h.transpose(1, 2), dim=1)
    out = F.silu(F.conv1d(u, w.unsqueeze(1), bias, padding=15, groups=Ci)).transpose(1, 2)
    gh, gw, gb = torch.autograd.grad(out, (h, w, bias), gout.double())
    return gh, torch.cat([gw, gb.unsqueeze(1)], dim=1)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("emu") / "libemu_u2c_glu_bwd.so")
    cmd = ["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-Wno-unknown-pragmas",
           "-o", so, os.path.join(HERE, "emu", "emu_u2c_glu_bwd.cpp")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    lib = ctypes.CDLL(so)
    fp = ctypes.POINTER(ctypes.c_float)
    lib.emu_u2c_glu_bwd.argtypes = [fp] * 6 + [ctypes.c_int] * 3

    def run(h, w, bias, gout):
        B, T, Ci = gout.shape
        arrs = [np.ascontiguousarray(t.numpy(), np.float32) for t in (h, w, bias, gout)]
        gh, dwb = np.full((B, T, 2 * Ci), np.nan, np.float32), np.full((Ci, 32), np.nan, np.float32)
        assert lib.emu_u2c_glu_bwd(*[a.ctypes.data_as(fp) for a in arrs + [gh, dwb]], B, T, Ci) == 0
        return torch.from_numpy(gh), torch.from_numpy(dwb)

    return run


# T = 20: shorter than the filter (padding on both sides of every frame); 64 / 65: exactly one tile / one frame into
# the second; 150: three tiles, the last one partial, halos crossing tile boundaries in both directions
@pytest.mark.parametrize("B,T,Ci", [(2, 20, 128), (1, 64, 128), (1, 65, 128), (2, 150, 256)])
def test_glu_backward_kernel_source_matches_float64_autograd(emu, B, T, Ci):
    g = torch.Generator().manual_seed(T)
    h, gout = torch.randn(B, T, 2 * Ci, generator=g), torch.randn(B, T, Ci, generator=g)
    w, bias = 0.2 * torch.randn(Ci, 31, generator=g), 0.2 * torch.randn(Ci, generator=g)
    gh, dwb = emu(h, w, bias, gout)
    want_gh, want_dwb = glu_dwconv_silu_reference(h, w, bias, gout)
    assert torch.isfinite(gh).all() and torch.isfinite(dwb).all()
    assert util.rms(gh - want_gh) <= 2e-6 * util.rms(want_gh)
    assert util.rms(dwb - want_dwb) <= 2e-6 * util.rms(want_dwb)
    assert (gh - want_gh).abs().max() <= 2e-5 * want_gh.abs().max()


@needs_gxx
def test_glu_backward_kernel_source_has_no_shared_memory_race(tmp_path):
    exe = str(tmp_path / "tsan_u2c_glu_bwd")
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-pthread", "-Wno-unknown-pragmas", "-o", exe,
           os.path.join(HERE, "emu", "tsan_u2c_glu_bwd.cpp")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0 and "tsan" in proc.stderr.lower():
        pytest.skip("ThreadSanitizer runtime not available: " + proc.stderr.strip().splitlines()[-1])
    assert proc.returncode == 0, proc.stderr
    res = subprocess.run([exe], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66"))
    assert "ThreadSanitizer" not in res.stderr, res.stderr[-4000:]
    assert res.returncode == 0 and "done" in res.stdout


def test_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    p, big = 16, 1 << 40                                       # a non-null address; a workspace size that always suffices
    assert L.b2d_u2c_backward_workspace_bytes(0, 8, 512, 4100) == 0 and L.b2d_u2c_backward_workspace_bytes(2, 8, 512, 0) == 0
    # 24 x 172: the depthwise partials (24 utterances x 3 tiles x 512 channels x 32) outweigh the column-sum slabs
    assert L.b2d_u2c_backward_workspace_bytes(24, 172, 512, 4100) == max(24 * 3 * 512 * 32 * 4, 33 * 4100 * 4)
    glu = lambda **kw: L.b2d_u2c_glu_dwconv_silu_backward(*[{**dict(h=p, w=p, b=p, g=p, gh=p, dwb=p, B=1, T=8, Ci=256, K=31,
                                                                  ws=p, n=big, s=0), **kw}[k]
                                                            for k in ("h", "w", "b", "g", "gh", "dwb", "B", "T", "Ci", "K", "ws", "n", "s")])
    assert glu(h=0) == -1 and glu(dwb=0) == -1 and glu(ws=0) == -1
    assert glu(K=29) == -2 and glu(Ci=100) == -2 and glu(B=65536) == -2 and glu(T=0) == -2
    assert glu(n=1 * 256 * 32 * 4 - 1) == -5
    assert b"u2c_glu_dwconv_silu_backward" in L.b2d_last_error()
    assert L.b2d_u2c_colsum(0, 4, 4, p, p, big, 0) == -1 and L.b2d_u2c_colsum(p, 0, 4, p, p, big, 0) == -2
    assert L.b2d_u2c_colsum(p, 129, 4, p, p, 2 * 4 * 4 - 1, 0) == -5                         # two slabs of 128 tokens
    assert L.b2d_u2c_layernorm_backward(p, p, p, 1e-5, 4, 128, p, p, p, big, 0) == -2        # C != 256
    assert L.b2d_u2c_layernorm_backward(p, p, 0, 1e-5, 4, 256, p, p, p, big, 0) == -1
    assert L.b2d_u2c_layernorm_backward(p, p, p, 1e-5, 4, 256, p, p, p, 2 * 256 * 4 - 1, 0) == -5
    gn = lambda C=256, G=4, st=p, n=big: L.b2d_u2c_groupnorm_lrelu_backward(p, st, p, p, 1e-5, 0.01, p, 1, 8, C, G, p, p, p, n, 0)
    assert gn(C=128) == -2 and gn(G=3) == -2 and gn(st=0) == -1 and gn(n=100) == -5
    assert L.b2d_u2c_embed_backward(p, p, p, p, 0, 0, 8, p, p, p, big, 0) == -2              # B = 0 (aug_shift may be null)
    assert L.b2d_u2c_embed_backward(p, p, p, p, 0, 1, 8, 0, p, p, big, 0) == -1
    assert L.b2d_u2c_embed_backward(p, p, p, p, 0, 1, 8, p, p, p, 4 * 256 * 4 - 1, 0) == -5
    assert L.b2d_u2c_conv3_fold(p, 1, 0, 256, p, 0) == -2 and L.b2d_u2c_conv3_fold(0, 1, 8, 256, p, 0) == -1
