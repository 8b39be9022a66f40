"""csrc/diffusion.cu's kernel source (the WaveNet stages and the sampler update of the diffusion models) executed on the
CPU (tests/emu/host_emu.h) against the float64 oracle (tests/diffusion_oracle.py) and float64 restatements, race-checked
under ThreadSanitizer, plus the argument checks of the new C ABI entries (no device touched).  The kernels run on
hardware in tests/test_gpu_diffusion.py."""
import math

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib
from tests import diffusion_oracle
from tests.emu_harness import abi_call, assert_race_free, shared, tsan
from tests.test_emu_reflow import check_operand, f32, out_buffers, ptr


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return shared("emu_diffusion.cpp", tmp_path_factory)


def conv_operand(y, T):
    """[B T, 3 C] operand of y [B, T, C]: [y(t - 1) | y(t) | y(t + 1)], zero outside each utterance"""
    B, _, C = y.shape
    pad = np.zeros((B, T + 2, C))
    pad[:, 1:-1] = y
    return np.concatenate([pad[:, :-2], pad[:, 1:-1], pad[:, 2:]], axis=2).reshape(B * T, 3 * C)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("B,T", [(3, 1), (2, 2), (2, 7)])
def test_input_stage_writes_the_convolution_operand_per_utterance(emu, split, B, T):
    rng = np.random.default_rng(B * 10 + T + split)
    C = 16
    g, bias = f32(rng.standard_normal((B, T, C))), f32(rng.standard_normal(C))
    step = f32(rng.standard_normal((B, 2 * C)))                       # one row per utterance, layer 0's slice first
    h = np.full((B, T, C), np.nan, np.float32)
    hi, lo = out_buffers((B * T, 3 * C), split)
    assert emu.emu_df_layer(ptr(g), ptr(bias), ptr(h), None, 0, ptr(step), 2 * C, 1.0, B, T, C, ptr(hi), ptr(lo)) == 0
    want_h = np.maximum(g.astype(np.float64) + bias, 0)
    assert np.abs(h - want_h).max() <= 1e-6 * np.abs(want_h).max()
    check_operand(hi, lo, conv_operand(want_h + step[:, None, :C], T))


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("last", [False, True])
def test_residual_stage(emu, split, stage, last):
    rng = np.random.default_rng(stage * 7 + split + 2 * last)
    B, T, C, L = 2, 5, 8, 3
    g, bias = f32(rng.standard_normal((B, T, 2 * C))), f32(rng.standard_normal(2 * C))
    h0, s0 = f32(rng.standard_normal((B, T, C))), f32(rng.standard_normal((B, T, C)))
    step = f32(rng.standard_normal((1, L * C)))
    h, skip = h0.copy(), s0.copy()
    shape = (B * T, C) if last else (B * T, 3 * C)
    hi, lo = out_buffers(shape, split)
    sp = None if last else step.ctypes.data + 4 * C                   # layer 1's slice, one row for every utterance
    assert emu.emu_df_layer(ptr(g), ptr(bias), ptr(h), ptr(skip), stage, sp, 0, math.sqrt(L), B, T, C, ptr(hi),
                            ptr(lo)) == 0
    r = g.astype(np.float64) + bias
    want_h = (h0 + r[..., :C]) / math.sqrt(2)
    want_s = r[..., C:] + (s0 if stage == 2 else 0)
    assert np.abs(h - want_h).max() <= 1e-6 * np.abs(want_h).max()
    assert np.abs(skip - want_s).max() <= 1e-6 * np.abs(want_s).max()
    if last:
        check_operand(hi, lo, want_s.reshape(B * T, C) / math.sqrt(L))
    else:
        check_operand(hi, lo, conv_operand(want_h + step[0, C:2 * C], T))


@pytest.mark.parametrize("split", [False, True])
def test_gate_and_relu(emu, split):
    rng = np.random.default_rng(3 + split)
    N, C, L = 11, 8, 2
    g = f32(3 * rng.standard_normal((N, 2 * C)))
    cond = f32(rng.standard_normal((N, L * 2 * C)))
    hi, lo = out_buffers((N, C), split)
    assert emu.emu_df_gate(ptr(g), cond.ctypes.data + 4 * 2 * C, L * 2 * C, N, C, ptr(hi), ptr(lo)) == 0
    z = g.astype(np.float64) + cond[:, 2 * C:]
    check_operand(hi, lo, 1 / (1 + np.exp(-z[:, :C])) * np.tanh(z[:, C:]), rel=2e-6)
    bias = f32(rng.standard_normal(C))
    hi, lo = out_buffers((N, C), split)
    assert emu.emu_df_relu(ptr(g[:, :C].copy()), ptr(bias), N, C, ptr(hi), ptr(lo)) == 0
    check_operand(hi, lo, np.maximum(g[:, :C].astype(np.float64) + bias, 0))


def test_one_evaluation_of_the_emulated_stages_matches_the_oracle_wavenet(emu):
    """the stages of csrc/diffusion.cu chained around float64 GEMMs (numpy) as ddsp_svc_b200.WaveNet._velocity chains
    them, against diffusion_oracle.WaveNet in float64: B = 3 with T = 1 for one utterance's neighbours"""
    torch.manual_seed(0)
    M, Hd, C, L, B, T = 16, 12, 8, 3, 3, 4
    net = diffusion_oracle.seeded_weights(diffusion_oracle.WaveNet(M, L, C, Hd), 5).double()
    rng = np.random.default_rng(9)
    for T in (1, 4):
        x, cond = rng.standard_normal((B, M, T)), rng.standard_normal((B, Hd, T))
        steps = np.array([3.5, 250.0, 999.0])
        with torch.no_grad():
            want = net(torch.from_numpy(x)[:, None], torch.from_numpy(steps).float(), torch.from_numpy(cond))[:, 0].numpy()
            e = net.mlp(net.diffusion_embedding(torch.from_numpy(steps).float(), torch.float64))
            srow = np.concatenate([Ly.diffusion_projection(e).numpy() for Ly in net.residual_layers], axis=1)
        w = lambda conv: conv.weight.detach().numpy()[:, :, 0]
        crow = np.concatenate([cond.transpose(0, 2, 1).reshape(B * T, Hd) @ w(Ly.conditioner_projection).T +
                               Ly.conditioner_projection.bias.detach().numpy() + Ly.dilated_conv.bias.detach().numpy()
                               for Ly in net.residual_layers], axis=1)
        xs = x.transpose(0, 2, 1).reshape(B * T, M)
        h, skip = np.zeros((B * T, C), np.float32), np.zeros((B * T, C), np.float32)
        us, vs = np.zeros((B * T, 3 * C), np.float32), np.zeros((B * T, C), np.float32)
        srow, crow = f32(srow), f32(crow)
        emu.emu_df_layer(ptr(f32(xs @ w(net.input_projection).T)), ptr(f32(net.input_projection.bias.detach())), ptr(h),
                         None, 0, ptr(srow), srow.shape[1], 1.0, B, T, C, ptr(us), None)
        for i, Ly in enumerate(net.residual_layers):
            cw = Ly.dilated_conv.weight.detach().numpy().transpose(0, 2, 1).reshape(2 * C, 3 * C)
            emu.emu_df_gate(ptr(f32(us.astype(np.float64) @ cw.T)), crow.ctypes.data + 4 * i * 2 * C, crow.shape[1],
                            B * T, C, ptr(vs), None)
            last = i + 1 == L
            emu.emu_df_layer(ptr(f32(vs.astype(np.float64) @ w(Ly.output_projection).T)),
                             ptr(f32(Ly.output_projection.bias.detach())), ptr(h), ptr(skip), 1 if i == 0 else 2,
                             None if last else srow.ctypes.data + 4 * (i + 1) * C, srow.shape[1], math.sqrt(L), B, T, C,
                             ptr(vs if last else us), None)
        out = np.zeros((B * T, C), np.float32)
        emu.emu_df_relu(ptr(f32(vs.astype(np.float64) @ w(net.skip_projection).T)), ptr(f32(net.skip_projection.bias.detach())),
                        B * T, C, ptr(out), None)
        got = (out.astype(np.float64) @ w(net.output_projection).T + net.output_projection.bias.detach().numpy())
        got = got.reshape(B, T, M).transpose(0, 2, 1)
        assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max(), (T, np.abs(got - want).max() / np.abs(want).max())


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("inplace", [False, True])
def test_update_kernel_forms_the_linear_combination(emu, split, inplace):
    rng = np.random.default_rng(20 + split + 2 * inplace)
    B, T, M = 2, 7, 12
    N = B * T
    g, bias, x0 = f32(rng.standard_normal((N, M))), f32(rng.standard_normal(M)), f32(rng.standard_normal((N, M)))
    hs = [f32(rng.standard_normal((N, M))) for _ in range(3)]
    noise = f32(rng.standard_normal((B, 1, M, T)))
    coef = f32([0.8, -0.3, 1.2, 0.45, -0.2, 0.15, 0.05, 0.6])
    x, h0 = x0.copy(), [h.copy() for h in hs]
    d_out = h0[2] if inplace else np.full((N, M), np.nan, np.float32)     # d written over the oldest history entry
    x_out = x if inplace else np.full((N, M), np.nan, np.float32)
    hi, lo = out_buffers((N, M), split)
    assert emu.emu_df_update(ptr(g), ptr(bias), ptr(coef), ptr(x), ptr(d_out), ptr(h0[0]), ptr(h0[1]), ptr(h0[2]),
                             ptr(noise), B, T, M, ptr(x_out), ptr(hi), ptr(lo)) == 0
    c = coef.astype(np.float64)
    eps = g.astype(np.float64) + bias
    d = c[0] * x0 + c[1] * eps
    want = c[2] * x0 + c[3] * d + c[4] * hs[0] + c[5] * hs[1] + c[6] * hs[2] + c[7] * noise[:, 0].transpose(0, 2, 1).reshape(N, M)
    assert np.abs(d_out - d).max() <= 1e-6 * np.abs(d).max()
    assert np.abs(x_out - want).max() <= 2e-6 * np.abs(want).max()
    check_operand(hi, lo, want, rel=2e-6)
    # without history, noise, outputs: only the operand
    hi2, _ = out_buffers((N, M), False)
    x2 = x0.copy()
    assert emu.emu_df_update(ptr(g), ptr(bias), ptr(coef), ptr(x2), None, None, None, None, None, B, T, M, None, ptr(hi2),
                             None) == 0
    assert np.array_equal(x2, x0)
    want2 = c[2] * x0 + c[3] * (c[0] * x0 + c[1] * eps)
    assert np.abs(hi2 - want2).max() <= 2e-6 * np.abs(want2).max()


def test_diffusion_kernel_source_has_no_race(tmp_path):
    assert_race_free(tsan("tsan_diffusion.cpp", tmp_path))


def test_diffusion_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    p = 16                                                     # a non-null, 16-byte aligned address
    ok = dict(g=p, bias=p, h=p, skip=p, stage=1, step=p, step_stride=0, skip_div=1.0, B=1, T=8, C=512, hi=p, lo=0, stream=0)
    layer = lambda **kw: abi_call("b2d_df_layer", dict(ok, **kw))
    assert layer(g=0) == -1 and layer(hi=0) == -1 and layer(skip=0) == -1 and layer(h=0) == -1
    assert layer(B=0) == -2 and layer(step_stride=100) == -2 and layer(step=0, skip_div=0.0) == -2
    assert layer(stage=3) == -4 and layer(stage=0, step=0) == -4
    assert layer(C=510) == -3 and layer(g=p + 4) == -3 and layer(step=p + 4) == -3 and layer(step_stride=1026) == -3
    assert b"df_layer" in L.b2d_last_error()
    ok_gate = dict(g=p, cond=p, cond_stride=1024, n_tokens=8, C=512, hi=p, lo=0, stream=0)
    gate = lambda **kw: abi_call("b2d_df_gate", dict(ok_gate, **kw))
    assert gate(cond=0) == -1 and gate(hi=0) == -1 and gate(n_tokens=0) == -2 and gate(cond_stride=1000) == -2
    assert gate(C=510, cond_stride=1020) == -3 and gate(cond_stride=1026) == -3 and gate(cond=p + 4) == -3
    ok_relu = dict(g=p, bias=p, n_tokens=8, C=512, hi=p, lo=0, stream=0)
    relu = lambda **kw: abi_call("b2d_df_relu", dict(ok_relu, **kw))
    assert relu(bias=0) == -1 and relu(C=0) == -2 and relu(C=6) == -3
    ok_up = dict(g=p, bias=p, coef=p, x=p, d_out=0, h1=0, h2=0, h3=0, noise=0, B=1, T=8, M=128, x_out=p, hi=0, lo=p,
                 stream=0)
    up = lambda **kw: abi_call("b2d_df_update", dict(ok_up, **kw))
    assert up() == -1 and up(hi=p, coef=0) == -1 and up(hi=p, x=0) == -1 and up(hi=p, T=0) == -2
