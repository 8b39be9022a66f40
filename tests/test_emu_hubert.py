"""csrc/hubert.cu's kernels without a GPU: their source executed on the CPU (tests/emu/host_emu.h, with its warp model
and per-CTA static shared arrays) against float64 torch, then under AddressSanitizer.  The positional weights go through
the package's own packer (hubert.pack_posconv).  The kernels run on hardware in tests/test_gpu_units.py.

Bounds are per element, from the kernels' fp32 arithmetic: an FMA chain of n terms is within n 2^-24 of exact relative
to the sum of the magnitudes of its terms (`mag`); the exact-erf GELU has slope <= 1.13 and adds a few ulp of its
output.  Integer outputs (hb_align's row indices) are compared exactly."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import hubert
from tests.emu_harness import asan, shared

NAN = float("nan")
U = 2.0 ** -24


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return shared("emu_hubert.cpp", tmp_path_factory)


def _rand(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(*shape, generator=g, dtype=torch.float64)).float().double()


def _p(t):
    return None if t is None else t.data_ptr()


@pytest.mark.parametrize("N,pad,silent", [(400, 40, False), (1600, 40, False), (1600, 0, False), (1600, 40, True)])
def test_conv0_and_groupnorm(lib, N, pad, silent):
    """Conv1d(1 -> 512, k 10, s 5) of the zero-padded clip, rows past L0 zero, and GroupNorm(512, 512)'s scale / shift
    from the per-tile fp64 partial sums: a 10-term FMA chain per output, statistics of those fp32 values in fp64 (so
    the scale and shift are within a few 2^-24 of the float64 reference's; a silent clip has variance 0)"""
    B = 2
    L0 = hubert.feature_lengths(N, pad)[0]
    La, tiles = L0 + 3, (L0 + 3 + 63) // 64
    x = torch.zeros(B, N, dtype=torch.float64) if silent else _rand(B, N, seed=N + pad, scale=0.1)
    w = _rand(512, 1, 10, seed=1, scale=0.3)
    gamma, beta = _rand(512, seed=2), _rand(512, seed=3, scale=0.1)
    ref = F.conv1d(F.pad(x, (pad, pad))[:, None], w, stride=5)                      # [B, 512, L0]
    mag = F.conv1d(F.pad(x, (pad, pad))[:, None].abs(), w.abs(), stride=5)
    y = torch.full((B, La, 512), NAN)
    part = torch.full((B, tiles, 2, 512), NAN, dtype=torch.float64)
    xf, wf = x.float().contiguous(), w.float().reshape(512, 10).contiguous()
    assert lib.emu_hb_conv0(_p(xf), B, N, pad, _p(wf), L0, La, _p(y), _p(part)) == 0
    assert torch.equal(y[:, L0:], torch.zeros(B, 3, 512))
    got = y[:, :L0].double().transpose(1, 2)
    assert ((got - ref).abs() <= 10 * U * mag).all()
    scale, shift = torch.full((B, 512), NAN), torch.full((B, 512), NAN)
    gf, bf = gamma.float(), beta.float()
    assert lib.emu_hb_gn_finalize(_p(part), B, tiles, L0, _p(gf), _p(bf), 1e-5, _p(scale), _p(shift)) == 0
    mean, var = ref.mean(-1), ref.var(-1, unbiased=False)
    want_scale = gamma / (var + 1e-5).sqrt()
    want_shift = beta - mean * want_scale
    assert ((scale.double() - want_scale).abs() <= 1e-5 * want_scale.abs()).all()
    assert ((shift.double() - want_shift).abs() <= 1e-5 * (want_shift.abs() + (mean * want_scale).abs()) + 1e-7).all()


@pytest.mark.parametrize("T", [1, 2, 37, 129])
def test_posconv(lib, T):
    """Conv1d(768, 768, 128, padding 64, groups 16) with the last frame dropped, + bias, GELU; T = 129 crosses two
    64-frame tiles.  A 6144-term FMA chain per output.  B 2 at T <= 2 (the utterance offset), 1 above"""
    B = 2 if T <= 2 else 1
    x = _rand(B, T, 768, seed=T)
    w, b = _rand(768, 48, 128, seed=4, scale=(48 * 128) ** -0.5), _rand(768, seed=5, scale=0.1)
    pre = F.conv1d(x.transpose(1, 2), w, b, padding=64, groups=16)[..., :T]
    mag = F.conv1d(x.abs().transpose(1, 2), w.abs(), b.abs(), padding=64, groups=16)[..., :T]
    ref = F.gelu(pre).transpose(1, 2)
    y = torch.full((B, T, 768), NAN)
    xf, wp, bf = x.float().contiguous(), hubert.pack_posconv(w.float()), b.float()
    assert lib.emu_hb_posconv(_p(xf), B, T, _p(wp), _p(bf), _p(y)) == 0
    assert torch.isfinite(y).all()
    assert ((y.double() - ref).abs() <= 1.13 * 6150 * U * mag.transpose(1, 2) + 8 * U * ref.abs()).all()


def _attention_ref(qkv, T):
    B = qkv.shape[0]
    q, k, v = (qkv[..., i * 768:(i + 1) * 768].reshape(B, T, 12, 64).transpose(1, 2) for i in range(3))
    s = q @ k.transpose(-1, -2) / 8
    p = s.softmax(-1)
    S = ((q.abs() / 8) @ k.abs().transpose(-1, -2)).amax(-1, keepdim=True)   # the largest score's term magnitudes
    o = (p @ v).transpose(1, 2).reshape(B, T, 768)
    pv = (p @ v.abs()).transpose(1, 2).reshape(B, T, 768)
    return o, pv, S.transpose(1, 2).expand(B, T, 12, 64).reshape(B, T, 768)


@pytest.mark.parametrize("T,peaked", [(1, False), (2, False), (63, False), (64, False), (65, False), (130, False),
                                      (70, True)])
def test_attention(lib, T, peaked):
    """12 heads x 64, 64-key tiles with keys past T masked.  A score is a 64-term FMA chain: its absolute error
    (64 S 2^-24, S the magnitude sum of the largest score) scales every weight by exp of it, and the softmax sum and
    the weighted value sum add T + 64 roundings of P |v|.  The peaked case scales q and k by 6 (scores in the hundreds:
    the running max must rescale).  B 2 at T <= 2 (the utterance offset), 1 above"""
    B = 2 if T <= 2 else 1
    qkv = _rand(B, T, 3 * 768, seed=T + 7 * peaked, scale=0.5)
    if peaked:
        qkv[..., :1536] *= 6
    o, pv, S = _attention_ref(qkv, T)
    hi, lo = torch.full((B, T, 768), NAN), torch.full((B, T, 768), NAN)
    qf = qkv.float().contiguous()
    assert lib.emu_hb_attention(_p(qf), B, T, _p(hi), _p(lo)) == 0
    got = hi.double() + lo.double()
    assert torch.isfinite(got).all()
    bound = (64 * S * 1.01 + T + 80) * U * pv + 2.0 ** -22 * o.abs()
    assert ((got - o).abs() <= bound).all(), ((got - o).abs() - bound).max().item()


@pytest.mark.parametrize("ratio", [16000 / 44100 * 512 / 320, 16000 / 16000 * 160 / 320])
def test_align(lib, ratio):
    """Units_Encoder.encode's gather at a 44.1 kHz / hop 512 and a 16 kHz / hop 160 rate: the rows picked are exactly
    hubert.align_index's (float32 product, half to even, clamped to T - 1)"""
    B, T, C, n_frames = 2, 23, 8, 60
    units = torch.arange(B * T * C, dtype=torch.float32).reshape(B, T, C)
    out = torch.full((B, n_frames, C), NAN)
    assert lib.emu_hb_align(_p(units), B, T, C, ratio, n_frames, _p(out)) == 0
    idx = torch.from_numpy(hubert.align_index(n_frames, ratio, T))
    assert torch.equal(out, units[:, idx])


def test_kernels_under_address_sanitizer(tmp_path):
    """every input in a heap buffer of exactly its size: conv0 with and without the pad and its GroupNorm statistics,
    attention at T = 1 and 65, posconv at T = 2, align, act with and without the affine, ln at C 512 (GELU, padded
    rows) and in place at C 768"""
    res = asan("emu_hubert.cpp", tmp_path, "EMU_ASAN")
    assert res.returncode == 0 and "done 0" in res.stdout, res.stderr[-4000:]


@pytest.mark.parametrize("split", [True, False])
def test_act(lib, split):
    """GELU(x scale[b, c] + shift[b, c]) of [B, L, C] over a 3-CTA grid-stride loop, written as the GEMM operand: the
    TF32 (hi, lo) halves or fp32 in hi; and without the affine.  One fmaf, then erff and four fp32 operations: within
    8 2^-24 (|GELU| + |v|) (the last term where 1 + erf cancels); the split adds 2^-22 |GELU|, and hi is TF32"""
    B, L, C = 2, 5, 40
    x = _rand(B, L, C, seed=30)
    scale, shift = _rand(B, C, seed=31), _rand(B, C, seed=32)
    for affine in (True, False):
        v = x * scale[:, None] + shift[:, None] if affine else x
        ref = F.gelu(v)
        hi, lo = torch.full((B, L, C), NAN), (torch.full((B, L, C), NAN) if split else None)
        xf, sf, hf = x.float().contiguous(), scale.float(), shift.float()
        assert lib.emu_hb_act(_p(xf), B * L, C, L if affine else B * L, _p(sf) if affine else None,
                              _p(hf) if affine else None, _p(hi), _p(lo)) == 0
        got = hi.double() + (lo.double() if split else 0)
        bound = 8 * U * (ref.abs() + v.abs()) + (2.0 ** -22 * ref.abs() if split else 0)
        assert ((got - ref).abs() <= bound).all()
        if split:
            assert ((hi.view(torch.int32) & 0x1FFF) == 0).all()


@pytest.mark.parametrize("C,mode", [(512, "gelu"), (768, "y"), (768, "y_in_place")])
def test_ln(lib, C, mode):
    """LayerNorm(C) of rows gathered from [B, rows_per_b, C] (C 512: 3 padded rows per utterance dropped, GELU first),
    + y (C 768), and in place over x (h == x, rows_per_b = T).  11 rows per utterance: the last CTA's tail warps
    return.  Bound: the mean and variance are fp32 sums of NPL terms per lane and a 5-step butterfly, the output one
    fmaf; with rstd and gamma, |err| <= |gamma| rstd (NPL + 16) 2^-24 (|v - mean| + mean |v|) plus the GELU's
    8 2^-24 (|v| + |x|) through the same gain, and 2 ulp of the output"""
    B, T = 2, 11
    per_b = T + 3 if mode == "gelu" else T
    npl = C // 32
    x = _rand(B, per_b, C, seed=C, scale=3) + 1
    y = _rand(B * T, C, seed=C + 1) if mode != "gelu" else None
    g, b = _rand(C, seed=33).abs() + 0.5, _rand(C, seed=34)
    xin = x[:, :T].reshape(B * T, C)
    v = xin + y if y is not None else F.gelu(xin)
    mean, var = v.mean(-1, keepdim=True), v.var(-1, unbiased=False, keepdim=True)
    rstd = (var + 1e-5).rsqrt()
    ref = F.layer_norm(v, (C,), g, b, 1e-5)
    gain = g.abs() * rstd
    bound = gain * (npl + 16) * U * ((v - mean).abs() + v.abs().mean(-1, keepdim=True))
    if mode == "gelu":
        bound = bound + gain * 8 * U * (v.abs() + xin.abs())
    bound = bound + 2 * U * ref.abs()
    xf = x.float().contiguous()
    yf, gf, bf = (y.float().contiguous() if y is not None else None), g.float(), b.float()
    hi, lo = torch.full((B * T, C), NAN), torch.full((B * T, C), NAN)
    h = xf if mode == "y_in_place" else torch.full((B * T, C), NAN)
    assert lib.emu_hb_ln(_p(xf), _p(yf), B * T, T, per_b, C, int(mode == "gelu"), _p(gf), _p(bf), 1e-5, _p(h), _p(hi),
                         _p(lo)) == 0
    got = h.reshape(B * T, C).double()
    assert ((got - ref).abs() <= bound).all(), ((got - ref).abs() - bound).max().item()
    assert ((hi.double() + lo.double() - got).abs() <= 2.0 ** -22 * got.abs()).all()
