"""csrc/diffusion_bwd.cu's kernel source (the diffusion loss's input and the WaveNet denoiser's backward stages) executed
on the CPU (tests/emu/host_emu.h) against float64 restatements, on several grids (results must be bit-identical), plus
the argument checks of the new C ABI entries (no device touched).  The kernels run on hardware in
tests/test_gpu_diffusion_backward.py.  They use no shared memory and no barrier: every output element has one owner
thread, which the grid-independence checks exercise."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib
from tests.emu_harness import abi_call, shared
from tests.test_emu_reflow_backward import GRIDS, check_halves, f32, halves, nan, ptr


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return shared("emu_diffusion_bwd.cpp", tmp_path_factory)


@pytest.fixture(scope="module")
def emu_rf(tmp_path_factory):
    return shared("emu_reflow_bwd.cpp", tmp_path_factory)


def tables():
    ac = np.cumprod(1.0 - np.linspace(1e-4, 0.02, 1000))
    return f32(np.sqrt(ac)), f32(np.sqrt(1.0 - ac))


@pytest.mark.parametrize("split", [False, True])
def test_loss_input_kernel(emu, split):
    rng = np.random.default_rng(1)
    B, T, M = 3, 37, 24
    gt, noise = f32(rng.standard_normal((B, T, M)) * 3 - 5), f32(rng.standard_normal((B, T, M)))
    t = np.array([0, 999, 417], dtype=np.int64)
    sa, s1m = tables()
    results = []
    for ctas, threads in GRIDS:
        hi, lo = halves((B, T, M), True) if split else (nan((B, T, M)), None)
        emu.emu_df_loss_input(ctas, threads, ptr(gt), ptr(noise), ptr(t), ptr(sa), ptr(s1m), 1000, -12.0, 14.0, B, T, M,
                              ptr(hi), ptr(lo))
        results.append((hi, lo))
    x0 = ((gt.astype(np.float64) + 12) / 14) * 2 - 1
    want = sa[t][:, None, None].astype(np.float64) * x0 + s1m[t][:, None, None].astype(np.float64) * noise
    hi, lo = results[0]
    if split:
        check_halves(hi, lo, want)
    else:
        # the reference's fp32 association exactly: norm_spec, then extract(a) x0 + extract(b) noise, each rounded
        x32 = ((gt - np.float32(-12)) / np.float32(14)) * np.float32(2) - np.float32(1)
        assert np.array_equal(hi, sa[t][:, None, None] * x32 + s1m[t][:, None, None] * noise)
    for other in results[1:]:
        assert all(a is None or np.array_equal(a, b) for a, b in zip(results[0], other))
    # a step outside the schedule gives NaN, not a read outside the tables
    bad = np.array([0, 1000, -1], dtype=np.int64)
    out = np.zeros((B, T, M), np.float32)
    emu.emu_df_loss_input(3, 32, ptr(gt), ptr(noise), ptr(bad), ptr(sa), ptr(s1m), 1000, -12.0, 14.0, B, T, M, ptr(out), None)
    assert np.isfinite(out[0]).all() and np.isnan(out[1:]).all()


@pytest.mark.parametrize("split", [False, True])
def test_relu_and_mish_backward_kernels(emu, split):
    rng = np.random.default_rng(2 + split)
    rows, C = 37, 20
    gy, pre, bias = f32(rng.standard_normal((rows, C))), f32(3 * rng.standard_normal((rows, C))), f32(rng.standard_normal(C))
    pre[0, :4] = -bias[:4]                                       # x = 0 exactly: no gradient, as torch's ReLU
    x = torch.from_numpy(pre.astype(np.float64) + bias).requires_grad_(True)
    torch.relu(x).backward(torch.from_numpy(gy).double())
    xm = torch.from_numpy(np.concatenate([pre, f32([[25.0, -30.0, 19.9, 20.1] * 5])])).double().requires_grad_(True)
    gym = f32(rng.standard_normal(xm.shape))
    torch.nn.functional.mish(xm).backward(torch.from_numpy(gym).double())
    outs = []
    for ctas, threads in GRIDS:
        gx = nan((rows, C))
        hi, lo = halves((rows, C), split)
        emu.emu_df_relu_backward(ctas, threads, ptr(gy), ptr(pre), ptr(bias), rows, C, ptr(gx), ptr(hi), ptr(lo))
        check_halves(hi, lo, x.grad.numpy())
        gm = nan(xm.shape)
        mhi, mlo = halves(xm.shape, split)
        xin = f32(xm.detach().numpy())
        emu.emu_df_mish_backward(ctas, threads, ptr(gym), ptr(xin), xin.size, ptr(gm), ptr(mhi), ptr(mlo))
        check_halves(mhi, mlo, xm.grad.numpy(), rel=3e-6)
        outs.append((gx, gm))
    assert np.array_equal(outs[0][0], x.grad.numpy().astype(np.float32))
    assert np.abs(outs[0][1] - xm.grad.numpy()).max() <= 3e-6 * np.abs(xm.grad.numpy()).max()
    assert all(np.array_equal(a[0], outs[0][0]) and np.array_equal(a[1], outs[0][1]) for a in outs)


@pytest.mark.parametrize("split", [False, True])
def test_gate_backward_kernel(emu, split):
    rng = np.random.default_rng(4 + split)
    N, C, nL, layer = 29, 12, 3, 1
    Z2 = 2 * C * nL
    ga, g = f32(rng.standard_normal((N, C))), f32(2 * rng.standard_normal((N, 2 * C)))
    cond = f32(rng.standard_normal((N, Z2)))                     # every layer's rows; this layer's at column 2 C layer
    z = torch.from_numpy(g.astype(np.float64) + cond[:, 2 * C * layer:2 * C * (layer + 1)]).requires_grad_(True)
    (torch.sigmoid(z[:, :C]) * torch.tanh(z[:, C:])).backward(torch.from_numpy(ga).double())
    want = z.grad.numpy()
    outs = []
    for ctas, threads in GRIDS:
        gz = nan((N, Z2))
        zh, zl = halves((N, Z2), split)
        emu.emu_df_gate_backward(ctas, threads, ptr(ga), ptr(g), ptr(cond) + 4 * 2 * C * layer, Z2, N, C, layer, nL,
                                 ptr(gz), ptr(zh), ptr(zl))
        blk = slice(2 * C * layer, 2 * C * (layer + 1))
        assert np.isnan(np.delete(gz, np.r_[blk], axis=1)).all()         # only this layer's column block is written
        if split:
            check_halves(zh[:, blk], zl[:, blk], want, rel=2e-6)
        outs.append(gz[:, blk].copy())
    assert np.abs(outs[0] - want).max() <= 2e-6 * np.abs(want).max()
    assert all(np.array_equal(o, outs[0]) for o in outs)


def layer_backward_reference(gus, gh_top, gsk, skip_div, B, T, C):
    """float64: per layer i reversed, g_y = the adjoint of the [y(t-1) | y(t) | y(t+1)] gather inside each utterance,
    g_h = g_h' / sqrt 2 + g_y; g_R of layer i - 1 = [g_h / sqrt 2 | g_sk / skip_div]; the step sums of g_y"""
    nL = len(gus)
    gh = gh_top.astype(np.float64)
    grs, sums = {}, np.zeros((B, nL * C))
    for i in reversed(range(nL)):
        gu = gus[i].astype(np.float64).reshape(B, T, 3, C)
        gy = gu[:, :, 1].copy()
        gy[:, :-1] += gu[:, 1:, 0]
        gy[:, 1:] += gu[:, :-1, 2]
        gh = gh / np.sqrt(2) + gy.reshape(B * T, C)
        sums[:, i * C:(i + 1) * C] = gy.sum(axis=1)
        grs[i] = np.concatenate([gh / np.sqrt(2), gsk.astype(np.float64) / skip_div], axis=1)
    return gh, grs, sums


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("B,T", [(2, 70), (3, 1), (2, 2), (1, 37)])
def test_layer_backward_and_step_sums(emu, emu_rf, split, B, T):
    """three layers in reverse after the start call: g_h, each layer's next g_R and the step sums against float64;
    T = 1 and T = 2 put every tap of the convolution's adjoint at an utterance edge"""
    rng = np.random.default_rng(6 + split + T)
    C, nL, skip_div = 16, 3, np.float32(np.sqrt(3.0))
    N = B * T
    gus = [f32(rng.standard_normal((N, 3 * C))) for _ in range(nL)]
    gsk = f32(rng.standard_normal((N, C)))
    runs = []
    for ctas, threads in GRIDS:
        gh = nan((N, C))
        gr = nan((N, 2 * C))
        ghi, glo = halves((N, 2 * C), split)
        emu.emu_df_layer_backward(ctas, threads, None, ptr(gh), ptr(gsk), skip_div, B, T, C, nL - 1, nL, ptr(gr), ptr(ghi),
                                  ptr(glo), None)
        assert np.array_equal(gh, np.zeros((N, C), np.float32))
        assert np.array_equal(gr[:, :C], np.zeros((N, C), np.float32)) and np.array_equal(gr[:, C:], gsk / skip_div)
        part = nan(B * -(-T // emu.emu_df_slab()) * nL * C, np.float64)
        grs = {}
        for i in reversed(range(nL)):
            nxt = i > 0
            gr_i, hi_i, lo_i = (nan((N, 2 * C)),) + (halves((N, 2 * C), split) if nxt else (None, None))
            emu.emu_df_layer_backward(ctas, threads, ptr(gus[i]), ptr(gh), ptr(gsk), skip_div, B, T, C, i, nL,
                                      ptr(gr_i) if nxt else None, ptr(hi_i), ptr(lo_i), ptr(part))
            if nxt:
                grs[i] = (gr_i, hi_i, lo_i)
        gS = nan((B, nL * C))
        emu_rf.emu_rf_step_sums(ctas, threads, ptr(part), B, T, nL * C, ptr(gS))
        runs.append((gh, gS, grs))
    want_h, want_r, want_s = layer_backward_reference(gus, np.zeros((N, C)), gsk, float(skip_div), B, T, C)
    gh, gS, grs = runs[0]
    assert np.abs(gh - want_h).max() <= 1e-6 * np.abs(want_h).max()
    assert np.abs(gS - want_s).max() <= 1e-6 * np.abs(want_s).max()
    for i, (gr_i, hi_i, lo_i) in grs.items():
        # want_r[i] was formed from g_h after layer i; the kernel of layer i writes the g_R of layer i - 1 from it
        assert np.abs(gr_i - want_r[i]).max() <= 1e-6 * np.abs(want_r[i]).max()
        check_halves(hi_i, lo_i, want_r[i])
    for other in runs[1:]:
        assert np.array_equal(other[0], gh) and np.array_equal(other[1], gS)
        assert all(all(a is None or np.array_equal(a, b) for a, b in zip(other[2][i], grs[i])) for i in grs)


def test_diffusion_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    p = 256
    ok_li = dict(gt=p, noise=p, t=p, sqrt_ac=p, sqrt_1m_ac=p, n_steps=1000, spec_min=-12.0, spec_range=14.0, B=2, T=40,
                 M=128, hi=p, lo=0, stream=0)
    li = lambda **kw: abi_call("b2d_df_loss_input", dict(ok_li, **kw))
    assert li(gt=0) == -1 and li(t=0) == -1 and li(sqrt_ac=0) == -1 and li(sqrt_1m_ac=0) == -1 and li(hi=0) == -1
    assert li(B=0) == -2 and li(M=-1) == -2 and li(n_steps=0) == -2
    ok_rb = dict(gy=p, pre=p, bias=p, n_rows=8, C=512, gx=p, hi=0, lo=0, stream=0)
    rb = lambda **kw: abi_call("b2d_df_relu_backward", dict(ok_rb, **kw))
    assert rb(gy=0) == -1 and rb(bias=0) == -1 and rb(gx=0) == -1 and rb(lo=p) == -1 and rb(n_rows=0) == -2 and rb(C=0) == -2
    ok_mb = dict(gy=p, x=p, n=2048, gx=p, hi=0, lo=0, stream=0)
    mb = lambda **kw: abi_call("b2d_df_mish_backward", dict(ok_mb, **kw))
    assert mb(x=0) == -1 and mb(gx=0) == -1 and mb(lo=p) == -1 and mb(n=0) == -2
    ok_gb = dict(ga=p, g=p, cond=p, cond_stride=3 * 1024, n_tokens=80, C=512, layer=1, n_layers=3, gz=p, gz_hi=0, gz_lo=0,
                 stream=0)
    gb = lambda **kw: abi_call("b2d_df_gate_backward", dict(ok_gb, **kw))
    assert gb(ga=0) == -1 and gb(cond=0) == -1 and gb(gz=0) == -1 and gb(gz_lo=p) == -1
    assert gb(cond_stride=1000) == -2 and gb(layer=3) == -2 and gb(layer=-1) == -2 and gb(n_layers=0) == -2
    assert gb(n_tokens=0) == -2
    ws_n = L.b2d_rf_backward_workspace_bytes(2, 40, 3 * 128)
    ok_lb = dict(gu=p, gh=p, gsk=p, skip_div=1.7, B=2, T=40, C=128, layer=0, n_layers=3, gr=p, gr_hi=0, gr_lo=0, ws=p,
                 ws_bytes=ws_n, stream=0)
    lb = lambda **kw: abi_call("b2d_df_layer_backward", dict(ok_lb, **kw))
    assert lb(gh=0) == -1 and lb(gsk=0) == -1 and lb(ws=0) == -1 and lb(gr=0, gr_hi=p) == -1 and lb(gr_lo=p) == -1
    assert lb(layer=3) == -2 and lb(n_layers=0) == -2 and lb(C=0) == -2 and lb(skip_div=0.0) == -2
    assert lb(ws_bytes=ws_n // 2) == -5 and lb(T=200) == -5
    assert b"df_layer_backward" in L.b2d_last_error()
