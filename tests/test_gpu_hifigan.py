"""The NSF-HiFiGAN generator on the kernels (ddsp_svc_b200.Generator, csrc/hifigan.cu) against float64: every launch
kind of the 44.1 kHz vocoder, the whole generator against tests/hifigan_oracle.py, replays of the reference's goldens,
determinism and a forward free of device syncs.  Measured errors go to tests/report.py (B2D_PARITY_REPORT).

Bounds are relative RMS (and relative max) errors, 2.5 to 3 times the largest measured on an H100 80GB HBM3 at a 700 W
power limit (DESIGN.md section 4.16); the fp32 eager oracle under torch's defaults (cuDNN TF32) is recorded beside the
whole-generator cases for comparison."""
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import hifigan, ops
from tests import hifigan_oracle as ho
from tests import report
from tests.golden import make_golden_hifigan as mk

pytestmark = pytest.mark.gpu
DEV = "cuda"
# measured: one convolution <= 1.3e-6 RMS / 1.6e-6 max (C 256, k 11); post 1.7e-7, 3.4e-6 for its one-sample case; the
# generator <= 5.6e-6 / 6.6e-6 (the fp32 eager oracle: 6e-4 / 1.4e-3)
CONV_RMS, CONV_MAX = 4e-6, 5e-6
POST_RMS = POST_MAX = 1e-5
GEN_RMS, GEN_MAX = 1.5e-5, 2e-5


def _err(out, ref):
    out, ref = out.double().cpu(), ref.double().cpu()
    scale = ref.pow(2).mean().sqrt().item()
    return ((out - ref).pow(2).mean().sqrt().item() / scale, (out - ref).abs().max().item() / ref.abs().max().item())


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return scale * torch.randn(*shape, generator=g, dtype=torch.float64)


def _lrelu(x, on):
    return F.leaky_relu(x, 0.1) if on else x


def _generator(model):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen = hifigan.Generator(ho.config(mk.MODELS[model]["h"]))
    gen.load_state_dict(mk.seeded_state_dict(model), strict=True)
    return gen.eval()


@pytest.mark.parametrize("layout", ["channel_major", "token_major_view"])
@pytest.mark.parametrize("B,T", [(1, 1), (2, 37), (3, 300)])
def test_conv_pre(layout, B, T):
    w, b = _rand(512, 128, 7, seed=1, scale=0.03), _rand(512, seed=2, scale=0.1)
    x = _rand(B, 128, T, seed=3)
    ref = F.conv1d(x, w, b, padding=3).transpose(1, 2)
    xd = x.float().to(DEV) if layout == "channel_major" else x.float().transpose(1, 2).contiguous().to(DEV).transpose(1, 2)
    out = ops.hifigan_conv(xd.transpose(1, 2), hifigan.pack_conv(w.float().to(DEV)), b.float().to(DEV), 7, 1, 512, False)
    rel, mx = _err(out, ref)
    report.record("hifigan/conv_pre/%s/%dx%d" % (layout, B, T), rel_rms=rel, rel_max=mx)
    assert rel < CONV_RMS and mx < CONV_MAX, (rel, mx)


@pytest.mark.parametrize("C", [256, 128, 64, 32, 16])
@pytest.mark.parametrize("k", [3, 7, 11])
@pytest.mark.parametrize("d", [1, 3, 5])
def test_resblock_conv(C, k, d):
    """plain, + residual, and + residual + accum / 3 (the MRF sum's last launch), B = 2 across tile and utterance edges"""
    B, T = 2, 300
    w, b = _rand(C, C, k, seed=C + k, scale=1.0 / (C * k) ** 0.5), _rand(C, seed=d, scale=0.1)
    x, res, acc = _rand(B, T, C, seed=5), _rand(B, T, C, seed=6), _rand(B, T, C, seed=7)
    conv = F.conv1d(_lrelu(x, True).transpose(1, 2), w, b, padding=d * (k - 1) // 2, dilation=d).transpose(1, 2)
    wp, bd = hifigan.pack_conv(w.float().to(DEV)), b.float().to(DEV)
    xd, rd, ad = x.float().to(DEV), res.float().to(DEV), acc.float().to(DEV)
    cases = [("plain", dict(), conv), ("residual", dict(residual=rd), conv + res),
             ("mrf", dict(residual=rd, accum=ad, div=3.0), (acc + conv + res) / 3)]
    for name, kw, ref in cases:
        out = ops.hifigan_conv(xd, wp, bd, k, d, C, True, **kw)
        rel, mx = _err(out, ref)
        report.record("hifigan/resblock/C%d_k%d_d%d/%s" % (C, k, d, name), rel_rms=rel, rel_max=mx)
        assert rel < CONV_RMS and mx < CONV_MAX, (name, rel, mx)
    out = ops.hifigan_conv(xd, wp, bd, k, d, C, True, residual=rd, out=rd)          # in place over the residual
    assert _err(out, conv + res)[0] < CONV_RMS


# (C_in, C_out, u, noise stride s): the 44.1 kHz vocoder's five stages; noise_convs k = 2 s, padding s / 2 (k = 1 last)
STAGES = [(512, 256, 8, 64), (256, 128, 8, 8), (128, 64, 2, 4), (64, 32, 2, 2), (32, 16, 2, 1)]


@pytest.mark.parametrize("stage", range(5))
@pytest.mark.parametrize("B,T", [(1, 1), (2, 2), (3, 37)])
def test_transposed_conv_with_source(stage, B, T):
    Cin, Cout, u, s = STAGES[stage]
    nk, pad = (2 * s, s // 2) if stage < 4 else (1, 0)
    w, b = _rand(Cin, Cout, 2 * u, seed=stage, scale=1.0 / Cin ** 0.5), _rand(Cout, seed=9, scale=0.1)
    wn, bn = _rand(Cout, 1, nk, seed=10, scale=1.0 / nk ** 0.5), _rand(Cout, seed=11, scale=0.1)
    x, har = _rand(B, T, Cin, seed=12), torch.tanh(_rand(B, T * u * s, 1, seed=13))
    ref = (F.conv_transpose1d(_lrelu(x, True).transpose(1, 2), w, b, stride=u, padding=u // 2) +
           F.conv1d(har.transpose(1, 2), wn, bn, stride=s, padding=pad)).transpose(1, 2)
    out = ops.hifigan_conv(x.float().to(DEV), hifigan.pack_conv(hifigan.polyphase(w.float().to(DEV), u)),
                           b.float().to(DEV), 3, 1, u * Cout, True, up=u, source=har.float().to(DEV),
                           noise_w=wn.float().reshape(Cout, nk).to(DEV), noise_b=bn.float().to(DEV), noise_stride=s,
                           noise_pad=pad)
    assert out.shape == ref.shape
    rel, mx = _err(out, ref)
    report.record("hifigan/ups/%d/%dx%d" % (stage, B, T), rel_rms=rel, rel_max=mx)
    assert rel < CONV_RMS and mx < CONV_MAX, (rel, mx)


def _takes_128_rows(T, N, B):
    """hifigan_conv_launch's choice: BM = 128 unless 128-row tiles leave the grid under two CTAs per SM"""
    BN = 32 if N % 32 == 0 else 16
    return -(-T // 128) * (N // BN) * B >= 2 * torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("C,k,d", [(32, 11, 5), (16, 7, 3)])
def test_resblock_conv_on_the_128_row_tile(C, k, d):
    """B 2 and T long enough for <128, 32> (C 32) and <128, 16> (C 16), with a T % 128 tail and + residual"""
    B = 2
    T = 128 * (-(-2 * torch.cuda.get_device_properties(0).multi_processor_count // ((C // (32 if C % 32 == 0 else 16))
                                                                                  * B))) + 37
    assert _takes_128_rows(T, C, B)
    w, b = _rand(C, C, k, seed=C + k, scale=1.0 / (C * k) ** 0.5), _rand(C, seed=d, scale=0.1)
    x, res = _rand(B, T, C, seed=5), _rand(B, T, C, seed=6)
    ref = F.conv1d(_lrelu(x, True).transpose(1, 2), w, b, padding=d * (k - 1) // 2, dilation=d).transpose(1, 2) + res
    out = ops.hifigan_conv(x.float().to(DEV), hifigan.pack_conv(w.float().to(DEV)), b.float().to(DEV), k, d, C, True,
                           residual=res.float().to(DEV))
    rel, mx = _err(out, ref)
    report.record("hifigan/resblock_bm128/C%d_k%d_d%d/%d" % (C, k, d, T), rel_rms=rel, rel_max=mx)
    assert rel < CONV_RMS and mx < CONV_MAX, (rel, mx)


@pytest.mark.parametrize("stage", [3, 4])
def test_transposed_conv_on_the_128_row_tile(stage):
    """the last two stages (N = u C_out = 64, BN 32; 32, BN 32) at B 2 and T long enough for BM = 128"""
    Cin, Cout, u, s = STAGES[stage]
    nk, pad = (2 * s, s // 2) if stage < 4 else (1, 0)
    B, N = 2, u * Cout
    T = 128 * (-(-2 * torch.cuda.get_device_properties(0).multi_processor_count // ((N // 32) * B))) + 5
    assert _takes_128_rows(T, N, B)
    w, b = _rand(Cin, Cout, 2 * u, seed=stage, scale=1.0 / Cin ** 0.5), _rand(Cout, seed=9, scale=0.1)
    wn, bn = _rand(Cout, 1, nk, seed=10, scale=1.0 / nk ** 0.5), _rand(Cout, seed=11, scale=0.1)
    x, har = _rand(B, T, Cin, seed=12), torch.tanh(_rand(B, T * u * s, 1, seed=13))
    ref = (F.conv_transpose1d(_lrelu(x, True).transpose(1, 2), w, b, stride=u, padding=u // 2) +
           F.conv1d(har.transpose(1, 2), wn, bn, stride=s, padding=pad)).transpose(1, 2)
    out = ops.hifigan_conv(x.float().to(DEV), hifigan.pack_conv(hifigan.polyphase(w.float().to(DEV), u)),
                           b.float().to(DEV), 3, 1, N, True, up=u, source=har.float().to(DEV),
                           noise_w=wn.float().reshape(Cout, nk).to(DEV), noise_b=bn.float().to(DEV), noise_stride=s,
                           noise_pad=pad)
    rel, mx = _err(out, ref)
    report.record("hifigan/ups_bm128/%d/%dx%d" % (stage, B, T), rel_rms=rel, rel_max=mx)
    assert rel < CONV_RMS and mx < CONV_MAX, (rel, mx)


@pytest.mark.parametrize("B,T", [(1, 1), (2, 4096), (3, 5000)])
def test_post(B, T):
    w, b = _rand(1, 16, 7, seed=14, scale=0.1), _rand(1, seed=15, scale=0.1)
    x = _rand(B, T, 16, seed=16)
    ref = torch.tanh(F.conv1d(F.leaky_relu(x.transpose(1, 2)), w, b, padding=3))
    out = ops.hifigan_post(x.float().to(DEV), w.float()[0].t().contiguous().to(DEV), b.float().to(DEV))
    rel, mx = _err(out, ref)
    report.record("hifigan/post/%dx%d" % (B, T), rel_rms=rel, rel_max=mx)
    assert out.shape == (B, 1, T) and rel < POST_RMS and mx < POST_MAX, (rel, mx)


def _inputs(B, nF, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.linspace(-8.0, 0.5, 128)[None, :, None] + 1.5 * torch.randn(B, 128, nF, generator=g)
    f0 = 100.0 + 300.0 * torch.rand(B, nF, generator=g)
    if nF > 1:
        f0[:, nF // 2] = 0.0
    noise = torch.randn(B, nF * 512, 9, generator=g)
    rand_ini = torch.rand(1, 1, 9, generator=g)
    rand_ini[..., 0] = 0
    return x, f0, rand_ini, noise


@pytest.mark.parametrize("B,nF", [(1, 172), (3, 37), (1, 1), (2, 2)])
def test_generator_against_float64(B, nF):
    gen = _generator("full").to(DEV)
    x, f0, rand_ini, noise = _inputs(B, nF, 100 + nF)
    with torch.no_grad():
        args = (x.to(DEV), f0.to(DEV), rand_ini.to(DEV), noise.to(DEV))
        out = gen(*args)
        har = gen.m_source(f0.to(DEV), gen.upp, rand_ini.to(DEV), noise.to(DEV))
        sd = mk.seeded_state_dict("full")
        ref = ho.build(ho.config(ho.FULL), sd, fold_dtype=torch.float32)(x.double(), har.cpu().double())
        eager = ho.build(ho.config(ho.FULL), sd, torch.float32).to(DEV)(x.to(DEV), har)
    assert out.shape == (B, 1, nF * 512)
    rel, mx = _err(out, ref)
    e_rel, e_mx = _err(eager, ref)
    report.record("hifigan/generator/%dx%d" % (B, nF), rel_rms=rel, rel_max=mx, eager_rel_rms=e_rel,
                  eager_rel_max=e_mx)
    assert rel < GEN_RMS and mx < GEN_MAX, (rel, mx)


@pytest.mark.parametrize("name", list(mk.CASES))
def test_golden_replay(name):
    c = mk.CASES[name]
    d = np.load(mk.path(name))
    gen = _generator(c["model"])
    if not c.get("weight_norm"):
        gen.remove_weight_norm()
    gen = gen.to(DEV)
    t = lambda k: torch.from_numpy(d[k]).to(DEV)
    with torch.no_grad():
        rand_ini, noise = mk.draws(d)
        out = gen(t("x"), t("f0"), rand_ini.to(DEV), noise.to(DEV))
    ref, ref32 = torch.from_numpy(d["out64"]), torch.from_numpy(d["out32"])
    rel, mx = _err(out, ref)
    r_rel, r_mx = _err(ref32, ref)
    report.record("hifigan/golden/" + name, rel_rms=rel, rel_max=mx, ref32_rel_rms=r_rel, ref32_rel_max=r_mx)
    # the source kernel's fp32 sines are part of this error (the float64 replay recomputes them)
    assert rel < GEN_RMS and mx < GEN_MAX, (rel, mx)


def test_two_calls_are_bit_identical_and_a_warm_forward_does_not_sync():
    gen = _generator("full").to(DEV)
    x, f0, rand_ini, noise = (v.to(DEV) for v in _inputs(3, 37, 7))
    xv = x.transpose(1, 2).contiguous().transpose(1, 2)          # NsfHifiGAN's mel.transpose(1, 2) view
    with torch.no_grad():
        a = gen(xv, f0, rand_ini, noise)
        b = gen(xv, f0, rand_ini, noise)
        assert torch.equal(a, b)
        assert torch.equal(gen(x, f0, rand_ini, noise), a)        # the strided conv_pre path gives the same bits
        n0 = ops.launches()
        torch.cuda.set_sync_debug_mode("error")
        try:
            gen(xv, f0, rand_ini, noise)
            gen(xv, f0)                                           # drawn rand_ini, in-kernel noise
        finally:
            torch.cuda.set_sync_debug_mode(0)
        per_call = (ops.launches() - n0) // 2
    report.record("hifigan/launches", per_call=per_call)
    # source (2: its frame scan and the sample kernel), conv_pre, 5 x (1 + 18), post
    assert per_call == 2 + 1 + 5 * 19 + 1
    torch.cuda.synchronize()
