"""csrc/unit2control_bwd.cu's GLU -> depthwise conv -> SiLU backward kernel source executed on the CPU
(tests/emu/host_emu.h) against autograd of the same op in float64, race-checked under ThreadSanitizer, plus the argument
checks of the new C ABI entries (no device touched).  The kernels run on hardware in
tests/test_gpu_unit2control_backward.py."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import _lib
from tests import util
from tests.emu_harness import abi_call, assert_race_free, shared, tsan


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
    lib = shared("emu_u2c_glu_bwd.cpp", tmp_path_factory)
    fp = ctypes.POINTER(ctypes.c_float)

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


def test_glu_backward_kernel_source_has_no_shared_memory_race(tmp_path):
    assert_race_free(tsan("tsan_u2c_glu_bwd.cpp", tmp_path))


def test_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    p, big = 16, 1 << 40                                       # a non-null address; a workspace size that always suffices
    assert L.b2d_u2c_backward_workspace_bytes(0, 8, 512, 4100) == 0 and L.b2d_u2c_backward_workspace_bytes(2, 8, 512, 0) == 0
    # 24 x 172: the depthwise partials (24 utterances x 3 tiles x 512 channels x 32) outweigh the column-sum slabs
    assert L.b2d_u2c_backward_workspace_bytes(24, 172, 512, 4100) == max(24 * 3 * 512 * 32 * 4, 33 * 4100 * 4)
    ok_glu = dict(h=p, weight=p, bias=p, gout=p, gh=p, dwb=p, B=1, T=8, inner_channels=256, kernel_size=31, ws=p,
                  ws_bytes=big, stream=0)
    glu = lambda **kw: abi_call("b2d_u2c_glu_dwconv_silu_backward", dict(ok_glu, **kw))
    assert glu(h=0) == -1 and glu(dwb=0) == -1 and glu(ws=0) == -1
    assert glu(kernel_size=29) == -2 and glu(inner_channels=100) == -2 and glu(B=65536) == -2 and glu(T=0) == -2
    assert glu(ws_bytes=1 * 256 * 32 * 4 - 1) == -5
    assert b"u2c_glu_dwconv_silu_backward" in L.b2d_last_error()
    assert L.b2d_u2c_colsum(0, 4, 4, p, p, big, 0) == -1 and L.b2d_u2c_colsum(p, 0, 4, p, p, big, 0) == -2
    assert L.b2d_u2c_colsum(p, 129, 4, p, p, 2 * 4 * 4 - 1, 0) == -5                         # two slabs of 128 tokens
    assert L.b2d_u2c_layernorm_backward(p, p, p, 1e-5, 4, 128, p, p, p, big, 0) == -2        # C != 256
    assert L.b2d_u2c_layernorm_backward(p, p, 0, 1e-5, 4, 256, p, p, p, big, 0) == -1
    assert L.b2d_u2c_layernorm_backward(p, p, p, 1e-5, 4, 256, p, p, p, 2 * 256 * 4 - 1, 0) == -5
    ok_gn = dict(x_pre=p, stats=p, gamma=p, beta=p, eps=1e-5, slope=0.01, gy=p, B=1, T=8, C=256, groups=4, gx=p,
                 dgamma_dbeta=p, ws=p, ws_bytes=big, stream=0)
    gn = lambda **kw: abi_call("b2d_u2c_groupnorm_lrelu_backward", dict(ok_gn, **kw))
    assert gn(C=128) == -2 and gn(groups=3) == -2 and gn(stats=0) == -1 and gn(ws_bytes=100) == -5
    assert L.b2d_u2c_embed_backward(p, p, p, p, 0, 0, 8, p, p, p, big, 0) == -2              # B = 0 (aug_shift may be null)
    assert L.b2d_u2c_embed_backward(p, p, p, p, 0, 1, 8, 0, p, p, big, 0) == -1
    assert L.b2d_u2c_embed_backward(p, p, p, p, 0, 1, 8, p, p, p, 4 * 256 * 4 - 1, 0) == -5
    assert L.b2d_u2c_conv3_fold(p, 1, 0, 256, p, 0) == -2 and L.b2d_u2c_conv3_fold(0, 1, 8, 256, p, 0) == -1
