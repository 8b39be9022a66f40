"""csrc/pcmer_bwd.cu's kernel sources (the PCmer attention backward) executed on the CPU (tests/emu/host_emu.h plus the
driver's warp-shuffle shim) against float64 autograd of the same ops, plus the argument checks of their C ABI entries (no
device touched).  The kernels use neither shared memory nor barriers, so they have no ThreadSanitizer driver.  They run
on hardware in tests/test_gpu_u2c_pcmer_backward.py."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib
from tests import util

HERE = os.path.dirname(os.path.abspath(__file__))
EPS = 1e-4


def features(dd, x, is_query, eps=EPS):
    """the forward's feature map (csrc/unit2control.cu, u2c_softmax_feat_kernel) as a torch expression of the projected
    rows dd [R, J] and the data rows x [R, 64]; float64 inputs give the float64 reference, with autograd through the max"""
    J = dd.shape[-1]
    diag = (x ** 2).sum(-1, keepdim=True) / 2 * (64 ** -0.5)
    if is_query:
        return J ** -0.5 * (torch.exp(dd - diag - dd.max(-1, keepdim=True).values) + eps)
    return J ** -0.5 * torch.exp(dd - diag + eps)


def features_backward_reference(g, dd, x, vec, scal, T, is_query):
    """float64 autograd: the cotangent g + scal vec[row / T] (queries) or g + vec[row / T] (keys) of the features ->
    (g_dd, g_x)"""
    dd, x = (t.double().requires_grad_(True) for t in (dd, x))
    full = g.double() + (scal.double().unsqueeze(1) if is_query else 1.0) * vec.double().repeat_interleave(T, dim=0)
    return torch.autograd.grad(features(dd, x, is_query), (dd, x), full)


def readout_backward_reference(g_out, out, d_inv):
    """[B, T, H, 64] token-major g_out, out; d_inv [B, H, T] -> [B, H, T, 65]: g_out d_inv | -(g_out . out) d_inv"""
    g, o = g_out.double().permute(0, 2, 1, 3), out.double().permute(0, 2, 1, 3)
    di = d_inv.double().unsqueeze(-1)
    return torch.cat([g * di, -(g * o).sum(-1, keepdim=True) * di], dim=-1)


def qkv_gather_reference(gq, gk, gv, qkv, normalized):
    """head-major g_q, g_k, g_v [B, H, T, 64] (cotangents of q / (|q| + 1e-8), k / (|k| + 1e-8) when normalized, with
    q, k from qkv [B, T, 3, H, 64]) -> g_qkv [B, T, 3, H, 64]"""
    out = []
    for i, g in enumerate((gq, gk, gv)):
        x = qkv[:, :, i].permute(0, 2, 1, 3).double().requires_grad_(True)
        y = x / (x.norm(dim=-1, keepdim=True) + 1e-8) if normalized and i < 2 else x
        out.append(torch.autograd.grad(y, x, g.double())[0].permute(0, 2, 1, 3))
    return torch.stack(out, dim=2)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("emu") / "libemu_u2c_pcmer_bwd.so")
    cmd = ["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-pthread", "-Wno-unknown-pragmas",
           "-o", so, os.path.join(HERE, "emu", "emu_u2c_pcmer_bwd.cpp")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    lib = ctypes.CDLL(so)
    fp, i = ctypes.POINTER(ctypes.c_float), ctypes.c_int
    lib.emu_attn_readout_bwd.argtypes = [fp] * 3 + [i] * 3 + [fp]
    lib.emu_feat_bwd.argtypes = [fp] * 5 + [i] * 4 + [ctypes.c_float, fp]
    lib.emu_qkv_gather_bwd.argtypes = [fp] * 4 + [i] * 4 + [fp]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _np(t):
    return np.ascontiguousarray(t.numpy(), np.float32)


def _rel(got, want):
    return util.rms(got.double() - want) / util.rms(want)


@pytest.mark.parametrize("B,H,T", [(2, 3, 5), (1, 8, 13)])              # 30 rows: the last CTA is partial
def test_readout_backward_kernel_source(emu, B, H, T):
    g = torch.Generator().manual_seed(T)
    g_out, out = torch.randn(B, T, H, 64, generator=g), torch.randn(B, T, H, 64, generator=g)
    d_inv = 0.1 + torch.rand(B, H, T, generator=g)
    a, o, d = _np(g_out), _np(out), _np(d_inv)
    gn = np.full((B, H, T, 65), np.nan, np.float32)
    assert emu.emu_attn_readout_bwd(_p(a), _p(o), _p(d), B, H, T, _p(gn)) == 0
    assert _rel(torch.from_numpy(gn), readout_backward_reference(g_out, out, d_inv)) <= 2e-7


def _feature_case(R, T, J, is_query, seed, tie=False):
    g = torch.Generator().manual_seed(seed)
    dd, x = 2.0 * torch.randn(R, J, generator=g), 0.5 * torch.randn(R, 64, generator=g)
    if tie:
        # row 0: a near-tie BEFORE the maximum (index 3 sits 1e-5 below index J - 5); row 1: the maximum at index 0
        dd[0, J - 5] = dd[0].max() + 0.5
        dd[0, 3] = dd[0, J - 5] - 1e-5
        dd[1, 0] = dd[1].max() + 0.25
    phi = features(dd, x, is_query)                                          # fp32, the forward's saved features
    gphi = torch.randn(R, J, generator=g)
    vec = torch.rand(R // T, J, generator=g) * (5.0 if is_query else 1.0)
    scal = torch.randn(R, generator=g)
    return dd, x, phi, gphi, vec, scal


@pytest.mark.parametrize("is_query", [1, 0])
@pytest.mark.parametrize("R,T,J", [(21, 7, 266), (16, 16, 266), (9, 3, 288), (8, 8, 33)])
def test_feature_backward_kernel_source(emu, is_query, R, T, J):
    dd, x, phi, gphi, vec, scal = _feature_case(R, T, J, is_query, seed=R + J, tie=is_query == 1)
    g, gx = _np(gphi).copy(), np.full((R, 64), np.nan, np.float32)
    assert emu.emu_feat_bwd(_p(g), _p(_np(phi)), _p(_np(x)), _p(_np(vec)), _p(_np(scal)), R, T, J, is_query, EPS, _p(gx)) == 0
    want_dd, want_x = features_backward_reference(gphi, dd, x, vec, scal, T, is_query)
    g, gx = torch.from_numpy(g), torch.from_numpy(gx)
    assert torch.isfinite(g).all() and torch.isfinite(gx).all()
    assert _rel(g, want_dd) <= 2e-6 and _rel(gx, want_x) <= 2e-6
    # every row on its own (a misplaced maximum would show as one bad row among many good ones)
    for r in range(R):
        assert _rel(g[r], want_dd[r]) <= 2e-6, r
    if is_query:                                                              # the maximum's term lands on the true maximum
        assert abs(g[0, J - 5].item() - want_dd[0, J - 5].item()) <= 1e-5 * want_dd[0].abs().max().item()
        assert abs(g[1, 0].item() - want_dd[1, 0].item()) <= 1e-5 * want_dd[1].abs().max().item()


def test_feature_backward_without_the_maximum_term_is_wrong(emu):
    """negative control of the test above: the float64 gradient with the row maximum detached differs from the kernel's"""
    R, T, J = 21, 7, 266
    dd, x, phi, gphi, vec, scal = _feature_case(R, T, J, 1, seed=R + J, tie=True)
    g, gx = _np(gphi).copy(), np.zeros((R, 64), np.float32)
    assert emu.emu_feat_bwd(_p(g), _p(_np(phi)), _p(_np(x)), _p(_np(vec)), _p(_np(scal)), R, T, J, 1, EPS, _p(gx)) == 0
    d64, x64 = dd.double().requires_grad_(True), x.double()
    diag = (x64 ** 2).sum(-1, keepdim=True) / 2 * 0.125
    phi64 = J ** -0.5 * (torch.exp(d64 - diag - d64.max(-1, keepdim=True).values.detach()) + EPS)
    full = gphi.double() + scal.double().unsqueeze(1) * vec.double().repeat_interleave(T, dim=0)
    wrong, = torch.autograd.grad(phi64, d64, full)
    assert _rel(torch.from_numpy(g), wrong) > 1e-3


@pytest.mark.parametrize("normalized", [0, 1])
@pytest.mark.parametrize("B,H,T", [(2, 3, 5), (1, 8, 9)])
def test_qkv_gather_backward_kernel_source(emu, normalized, B, H, T):
    g = torch.Generator().manual_seed(T + normalized)
    gq, gk, gv = (torch.randn(B, H, T, 64, generator=g) for _ in range(3))
    qkv = torch.randn(B, T, 3, H, 64, generator=g) * 3.0
    out = np.full((B, T, 3, H, 64), np.nan, np.float32)
    assert emu.emu_qkv_gather_bwd(_p(_np(gq)), _p(_np(gk)), _p(_np(gv)), _p(_np(qkv)), B, H, T, normalized, _p(out)) == 0
    want = qkv_gather_reference(gq, gk, gv, qkv, normalized)
    got = torch.from_numpy(out)
    assert _rel(got, want) <= 2e-6
    assert torch.equal(got[:, :, 2], gv.permute(0, 2, 1, 3))                   # v is a pure gather


def test_pcmer_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    p = 16                                                     # a non-null address
    ro = lambda **kw: L.b2d_u2c_attn_readout_backward(*[{**dict(g=p, o=p, d=p, B=1, H=8, T=4, dh=64, gn=p, s=0), **kw}[k]
                                                         for k in ("g", "o", "d", "B", "H", "T", "dh", "gn", "s")])
    assert ro(g=0) == -1 and ro(d=0) == -1 and ro(gn=0) == -1
    assert ro(dh=32) == -2 and ro(T=0) == -2 and ro(B=-1) == -2
    assert b"u2c_attn_readout_backward" in L.b2d_last_error()
    ft = lambda **kw: L.b2d_u2c_softmax_features_backward(*[{**dict(g=p, f=p, x=p, v=p, sc=p, R=8, T=4, J=266, dh=64, q=1, e=1e-4,
                                                                      gx=p, s=0), **kw}[k]
                                                            for k in ("g", "f", "x", "v", "sc", "R", "T", "J", "dh", "q", "e", "gx", "s")])
    assert ft(g=0) == -1 and ft(x=0) == -1 and ft(gx=0) == -1 and ft(sc=0) == -1
    assert ft(dh=65) == -2 and ft(J=289) == -2 and ft(R=9) == -2 and ft(R=0) == -2
    assert b"u2c_softmax_features_backward" in L.b2d_last_error()
    qg = lambda **kw: L.b2d_u2c_qkv_gather_backward(*[{**dict(q=p, k=p, v=p, x=p, B=1, H=8, T=4, dh=64, n=1, o=p, s=0), **kw}[k]
                                                      for k in ("q", "k", "v", "x", "B", "H", "T", "dh", "n", "o", "s")])
    assert qg(q=0) == -1 and qg(o=0) == -1 and qg(x=0) == -1
    assert qg(dh=128) == -2 and qg(H=0) == -2
    assert b"u2c_qkv_gather_backward" in L.b2d_last_error()
