"""csrc/reflow_bwd.cu's kernel source (the reflow loss, its backward and the velocity network's backward stages) executed
on the CPU (tests/emu/host_emu.h) against float64 restatements, on several grids (results must be bit-identical), plus
the argument checks of the new C ABI entries (no device touched).  The kernels run on hardware in
tests/test_gpu_reflow_backward.py.  They use no shared memory and no barrier, so no ThreadSanitizer driver is needed:
every output element has one owner thread, which the grid-independence checks exercise."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib
from tests.emu_harness import abi_call, shared

GRIDS = [(1, 32), (3, 32), (7, 64)]                # (CTAs, threads per CTA)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return shared("emu_reflow_bwd.cpp", tmp_path_factory)


def f32(a):
    return np.ascontiguousarray(np.asarray(a, np.float32))


def ptr(a):
    return None if a is None else a.ctypes.data


def nan(shape, dtype=np.float32):
    return np.full(shape, np.nan, dtype)


def halves(shape, split):
    return (nan(shape), nan(shape)) if split else (None, None)


def check_halves(hi, lo, want, rel=1e-6):
    """split halves: TF32-exact (low 13 mantissa bits zero) and hi + lo = the value to 2^-22"""
    if hi is None:
        return
    got = hi.astype(np.float64) + lo.astype(np.float64)
    assert np.abs(got - want).max() <= rel * np.abs(want).max()
    for part in (hi, lo):
        assert not (part.view(np.uint32) & 0x1FFF).any()


def slabs(emu, T):
    return -(-T // emu.emu_rf_slab())


def loss_case(seed, B=3, T=45, M=24):
    rng = np.random.default_rng(seed)
    t = f32(np.clip(rng.random(B), 1e-7, 1 - 1e-7))
    w = f32(0.398942 / t / (1 - t) * np.exp(-0.5 * np.log(t / (1 - t)) ** 2))
    return dict(gt=f32(rng.standard_normal((B, T, M)) * 3 - 5), x0=f32(rng.standard_normal((B, T, M))), t=t, w=w,
                g=f32(rng.standard_normal((B, T, M))), bias=f32(rng.standard_normal(M)),
                target=f32(rng.standard_normal((B, T, M))), B=B, T=T, M=M)


@pytest.mark.parametrize("split", [False, True])
def test_loss_input_kernel(emu, split):
    c = loss_case(1)
    B, T, M = c["B"], c["T"], c["M"]
    x1 = ((c["gt"].astype(np.float64) + 12) / 14) * 2 - 1
    want_target = x1 - c["x0"]
    want_xt = c["x0"] + c["t"][:, None, None].astype(np.float64) * want_target
    results = []
    for ctas, threads in GRIDS:
        target = nan((B, T, M))
        hi, lo = halves((B, T, M), True) if split else (nan((B, T, M)), None)
        emu.emu_rf_loss_input(ctas, threads, ptr(c["gt"]), ptr(c["x0"]), ptr(c["t"]), -12.0, 14.0, B, T, M, ptr(target),
                              ptr(hi), ptr(lo))
        results.append((target, hi, lo))
    target, hi, lo = results[0]
    assert np.abs(target - want_target).max() <= 1e-6 * np.abs(want_target).max()
    if split:
        check_halves(hi, lo, want_xt)
    else:
        assert np.abs(hi - want_xt).max() <= 1e-6 * np.abs(want_xt).max()
    # the reference's fp32 association exactly: x1, x1 - x0, x0 + t (x1 - x0), each rounded to fp32
    x1_32 = ((c["gt"] - np.float32(-12)) / np.float32(14)) * np.float32(2) - np.float32(1)
    d32 = x1_32 - c["x0"]
    assert np.array_equal(target, d32)
    if not split:
        assert np.array_equal(hi, c["x0"] + c["t"][:, None, None] * d32)
    for other in results[1:]:
        assert all(a is None or np.array_equal(a, b) for a, b in zip(results[0], other))


@pytest.mark.parametrize("T", [45, 32, 7])
def test_loss_kernel_against_float64_and_on_every_grid(emu, T):
    c = loss_case(2 + T, T=T)
    B, M = c["B"], c["M"]
    e = c["target"].astype(np.float64) - (c["g"].astype(np.float64) + c["bias"])
    want = (c["w"][:, None, None].astype(np.float64) * e * e).mean()
    losses = []
    for ctas, threads in GRIDS:
        part, cols, loss = nan(B * slabs(emu, T) * M, np.float64), nan(M, np.float64), nan(1)
        emu.emu_rf_loss(ctas, threads, ptr(c["g"]), ptr(c["bias"]), ptr(c["target"]), ptr(c["w"]), B, T, M, ptr(part),
                        ptr(cols), ptr(loss))
        losses.append(loss[0])
    assert abs(losses[0] - want) <= 1e-6 * abs(want)
    assert all(x.tobytes() == losses[0].tobytes() for x in losses)


@pytest.mark.parametrize("split", [False, True])
def test_loss_backward_kernel(emu, split):
    c = loss_case(3)
    B, T, M = c["B"], c["T"], c["M"]
    gl = f32([0.75])
    v = c["g"].astype(np.float64) + c["bias"]
    want = 0.75 * 2 * c["w"][:, None, None].astype(np.float64) * (v - c["target"]) / (B * T * M)
    outs = []
    for ctas, threads in GRIDS:
        gv = nan((B, T, M))
        hi, lo = halves((B, T, M), split)
        emu.emu_rf_loss_backward(ctas, threads, ptr(c["g"]), ptr(c["bias"]), ptr(c["target"]), ptr(c["w"]), ptr(gl), B, T, M,
                                 ptr(gv), ptr(hi), ptr(lo))
        outs.append((gv, hi, lo))
    gv, hi, lo = outs[0]
    assert np.abs(gv - want).max() <= 1e-6 * np.abs(want).max()
    check_halves(hi, lo, want)
    assert all(np.array_equal(a[0], outs[0][0]) for a in outs)
    # autograd of the loss expression in float64 agrees (the formula, not only the kernel's restatement)
    g64 = torch.from_numpy(c["g"]).double().requires_grad_(True)
    e = torch.from_numpy(c["target"]).double() - (g64 + torch.from_numpy(c["bias"]).double())
    (0.75 * (torch.from_numpy(c["w"]).double()[:, None, None] * e * e).mean()).backward()
    assert np.abs(g64.grad.numpy() - want).max() <= 1e-12 * np.abs(want).max()


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("with_bias", [False, True])
def test_gelu_backward_kernel(emu, split, with_bias):
    rng = np.random.default_rng(4 + split + 2 * with_bias)
    rows, C = 37, 20
    gy, pre = f32(rng.standard_normal((rows, C))), f32(3 * rng.standard_normal((rows, C)))
    bias = f32(rng.standard_normal(C)) if with_bias else None
    x = torch.from_numpy(pre.astype(np.float64) + (bias if with_bias else 0)).requires_grad_(True)
    torch.nn.functional.gelu(x).backward(torch.from_numpy(gy).double())
    want = x.grad.numpy()
    outs = []
    for ctas, threads in GRIDS:
        gx = nan((rows, C))
        hi, lo = halves((rows, C), split)
        emu.emu_rf_gelu_backward(ctas, threads, ptr(gy), ptr(pre), ptr(bias), rows, C, ptr(gx), ptr(hi), ptr(lo))
        outs.append(gx)
        check_halves(hi, lo, want, rel=2e-6)
    assert np.abs(outs[0] - want).max() <= 2e-6 * np.abs(want).max()
    assert all(np.array_equal(o, outs[0]) for o in outs)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("T", [70, 9])
def test_layer_backward_and_step_sums(emu, split, T):
    """two layers in reverse order: g_h accumulates both g_z, G_Z holds each in its column block, the step sums are the
    per-utterance token sums of G_Z"""
    rng = np.random.default_rng(5 + split + T)
    B, D, nL = 2, 40, 2
    LD, N = D * nL, B * T
    gzs = [f32(rng.standard_normal((N, D))) for _ in range(nL)]
    gh0 = f32(rng.standard_normal((N, D)))
    runs = []
    for ctas, threads in GRIDS:
        gh = gh0.copy()
        gh_hi, gh_lo = halves((N, D), split)
        z = nan((N, LD))
        z_hi, z_lo = halves((N, LD), split)
        part = nan(B * slabs(emu, T) * LD, np.float64)
        for i in reversed(range(nL)):
            emu.emu_rf_layer_backward(ctas, threads, ptr(gzs[i]), ptr(gh), B, T, D, i, nL, ptr(gh_hi), ptr(gh_lo), ptr(z),
                                      ptr(z_hi), ptr(z_lo), ptr(part))
            if i == 1:
                want_h = gh0.astype(np.float64) + gzs[1]
                assert np.abs(gh - want_h).max() <= 1e-6 * np.abs(want_h).max()
                check_halves(gh_hi, gh_lo, want_h)
        gS = nan((B, LD))
        emu.emu_rf_step_sums(ctas, threads, ptr(part), B, T, LD, ptr(gS))
        runs.append((gh, z, gS, gh_hi, z_hi, z_lo))
    gh, z, gS = runs[0][:3]
    want_h = gh0.astype(np.float64) + gzs[1] + gzs[0]
    want_z = np.concatenate(gzs, axis=1).astype(np.float64)
    assert np.abs(gh - want_h).max() <= 1e-6 * np.abs(want_h).max()
    assert np.array_equal(z, want_z.astype(np.float32))
    check_halves(runs[0][4], runs[0][5], want_z)
    want_s = want_z.reshape(B, T, LD).sum(axis=1)
    assert np.abs(gS - want_s).max() <= 1e-6 * np.abs(want_s).max()
    for other in runs[1:]:
        assert all(a is None or np.array_equal(a, b) for a, b in zip(runs[0], other))


def test_reflow_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    p = 256
    assert L.b2d_rf_backward_workspace_bytes(0, 8, 128) == 0 and L.b2d_rf_backward_workspace_bytes(2, 8, 0) == 0
    ws_n = L.b2d_rf_backward_workspace_bytes(2, 40, 128)
    assert ws_n >= 2 * 2 * 128 * 8 + 128 * 8
    ok_li = dict(gt=p, x0=p, t=p, spec_min=-12.0, spec_range=14.0, B=2, T=40, M=128, target=p, hi=p, lo=0, stream=0)
    li = lambda **kw: abi_call("b2d_rf_loss_input", dict(ok_li, **kw))
    assert li(gt=0) == -1 and li(t=0) == -1 and li(hi=0) == -1 and li(target=0) == -1 and li(B=0) == -2 and li(M=-1) == -2
    ok_loss = dict(g=p, bias=p, target=p, w=p, B=2, T=40, M=128, ws=p, ws_bytes=ws_n, loss=p, stream=0)
    loss = lambda **kw: abi_call("b2d_rf_loss", dict(ok_loss, **kw))
    assert loss(w=0) == -1 and loss(ws=0) == -1 and loss(loss=0) == -1 and loss(T=0) == -2
    assert loss(ws_bytes=ws_n - 8) == -5 and loss(T=80) == -5
    ok_lb = dict(g=p, bias=p, target=p, w=p, g_loss=p, B=2, T=40, M=128, gv=p, hi=0, lo=0, stream=0)
    lb = lambda **kw: abi_call("b2d_rf_loss_backward", dict(ok_lb, **kw))
    assert lb(g_loss=0) == -1 and lb(gv=0) == -1 and lb(lo=p) == -1 and lb(B=0) == -2
    ok_gb = dict(gy=p, pre=p, bias=0, n_rows=8, C=512, gx=p, hi=0, lo=0, stream=0)
    gb = lambda **kw: abi_call("b2d_rf_gelu_backward", dict(ok_gb, **kw))
    assert gb(gy=0) == -1 and gb(gx=0) == -1 and gb(lo=p) == -1 and gb(n_rows=0) == -2 and gb(C=0) == -2
    lay_n = L.b2d_rf_backward_workspace_bytes(2, 40, 3 * 128)
    ok_ly = dict(gz=p, gh=p, B=2, T=40, D=128, layer=0, n_layers=3, gh_hi=0, gh_lo=0, z=p, z_hi=0, z_lo=0, ws=p,
                 ws_bytes=lay_n, stream=0)
    ly = lambda **kw: abi_call("b2d_rf_layer_backward", dict(ok_ly, **kw))
    assert ly(gz=0) == -1 and ly(z=0) == -1 and ly(ws=0) == -1 and ly(gh_lo=p) == -1 and ly(z_lo=p) == -1
    assert ly(layer=3) == -2 and ly(layer=-1) == -2 and ly(n_layers=0) == -2 and ly(D=0) == -2
    assert ly(ws_bytes=lay_n // 2) == -5 and ly(T=200) == -5
    ok_ss = dict(ws=p, ws_bytes=lay_n, B=2, T=40, cols=384, out=p, stream=0)
    ss = lambda **kw: abi_call("b2d_rf_step_sums", dict(ok_ss, **kw))
    assert ss(ws=0) == -1 and ss(out=0) == -1 and ss(cols=0) == -2 and ss(cols=768) == -5
    assert b"rf_step_sums" in L.b2d_last_error()
