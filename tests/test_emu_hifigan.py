"""csrc/hifigan.cu's kernels without a GPU: their source executed on the CPU (tests/emu/host_emu.h, with its warp,
mma.sync and cp.async models) against float64 torch, at the tile, halo and utterance edges and for every <BM, BN>
instantiation of hg_conv (the GPU picks one per shape; here each runs at every shape), then under AddressSanitizer.
Weights go through the package's own packers (hifigan.pack_conv, hifigan.polyphase), so the packing is checked together
with the kernel code that reads the fragments.  The kernels run on hardware in tests/test_gpu_hifigan.py.

Bounds, per output element, from the arithmetic: the inputs and weights are fp32 values, so the float64 reference is
exact for them.  3xTF32 (hi hi + lo hi + hi lo) leaves each product within 3 2^-22 of exact (|x - hi - lo| <= 2^-22 |x|
for both operands, and the dropped lo lo term).  The emulated mma sums its 8 products exactly and rounds once to fp32,
and the kernel adds its results in fp32: 2 k mma results per 16-channel chunk, one rounded add per chunk, then bias,
residual, accumulator and the division.  Each rounding is within 2^-24 of a partial sum bounded by `mag`, the same
convolution of |x| and |w| plus |bias|, |residual| and |accum|.  So |out - ref| <= (3 2^-22 + (2 k + chunks + 4) 2^-24)
mag.  The relative RMS error must also stay under 1e-6, where the 3xTF32 kernels land."""
import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import hifigan
from tests.emu_harness import asan, shared

pytestmark = pytest.mark.filterwarnings("ignore")
INST = [(64, 32), (64, 16), (128, 32), (128, 16)]
REL_RMS = 1e-6


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return shared("emu_hifigan.cpp", tmp_path_factory)


def _rand(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(*shape, generator=g, dtype=torch.float64)).float().double()


def _p(t):
    return None if t is None else t.data_ptr()


def _check(out, ref, mag, steps):
    out = out.double()
    assert torch.isfinite(out).all(), "unwritten or poisoned elements"
    err = (out - ref).abs()
    bound = (3 * 2.0 ** -22 + (steps + 4) * 2.0 ** -24) * mag
    worst = (err - bound).max().item()
    assert worst <= 0, ("element bound exceeded", worst, err.max().item())
    rel = ((out - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    assert rel < REL_RMS, rel
    return rel


def _conv(lib, BM, BN, x, w, b, k, d, N, lrelu, residual=None, accum=None, div=1.0, out=None, strides=None, T=None):
    """x: fp32 [B, T, C], or a buffer read through `strides` (sb, st, sc) for T frames"""
    C = w.numel() // (2 * k * N)                  # the packed weight holds hi and lo of N C k values
    if strides is None:
        B, T_, _ = x.shape
        sb, st, sc = x.stride()
    else:
        B, T_ = x.shape[0], T
        sb, st, sc = strides
    out = torch.full((B, T_, N), float("nan")) if out is None else out
    rc = lib.emu_hg_conv(BM, BN, _p(x), sb, st, sc, B, T_, C, _p(w), _p(b), k, d, N, int(lrelu), _p(residual),
                         _p(accum), div, 0, None, None, None, 0, 0, 0, _p(out))
    assert rc == 0
    return out


LENGTHS = lambda BM, halo: [1, 2, BM - 1, BM, BM + 1, 2 * BM + halo]


@pytest.mark.parametrize("BM,BN", INST)
@pytest.mark.parametrize("Ti", range(6))
def test_conv_across_tile_and_utterance_edges(lib, BM, BN, Ti):
    """k 7, d 3 (a 9-row halo), C 32, B 3: T = 1, 2, BM - 1, BM, BM + 1 and 2 BM + halo"""
    C, k, d, B = 32, 7, 3, 3
    T = LENGTHS(BM, d * (k - 1) // 2)[Ti]
    w, b = _rand(C, C, k, seed=1, scale=(C * k) ** -0.5), _rand(C, seed=2, scale=0.1)
    x = _rand(B, T, C, seed=3)
    xl = F.leaky_relu(x, 0.1)
    ref = F.conv1d(xl.transpose(1, 2), w, b, padding=d * (k - 1) // 2, dilation=d).transpose(1, 2)
    mag = F.conv1d(xl.abs().transpose(1, 2), w.abs(), b.abs(), padding=d * (k - 1) // 2, dilation=d).transpose(1, 2)
    out = _conv(lib, BM, BN, x.float(), hifigan.pack_conv(w.float()), b.float(), k, d, C, True)
    _check(out, ref, mag, 2 * k + C // 16)


# (k, d, C): every kernel size, dilation and channel count of the 44.1 kHz vocoder's ResBlocks among them
SHAPES = [(3, 1, 16), (3, 5, 64), (7, 3, 32), (11, 1, 32), (11, 5, 16), (7, 5, 32), (3, 3, 32), (11, 3, 16)]


@pytest.mark.parametrize("i", range(len(SHAPES)))
def test_conv_variants(lib, i):
    """plain, + residual, the MRF sum (acc + conv + res) / 3 and in place over the residual, B 2, T BM + 1; the shapes
    take the four instantiations in turn (BN 16 where 32 does not divide C, as the launcher does)"""
    k, d, C = SHAPES[i]
    BM, BN = INST[i % 4] if C % 32 == 0 else INST[1 + 2 * (i % 2)]
    B, T, pad = 2, BM + 1, d * (k - 1) // 2
    w, b = _rand(C, C, k, seed=C + k, scale=(C * k) ** -0.5), _rand(C, seed=d, scale=0.1)
    x, res, acc = _rand(B, T, C, seed=5), _rand(B, T, C, seed=6), _rand(B, T, C, seed=7)
    xl = F.leaky_relu(x, 0.1)
    conv = F.conv1d(xl.transpose(1, 2), w, b, padding=pad, dilation=d).transpose(1, 2)
    mag = F.conv1d(xl.abs().transpose(1, 2), w.abs(), b.abs(), padding=pad, dilation=d).transpose(1, 2)
    wp, bf = hifigan.pack_conv(w.float()), b.float()
    xf, rf, af = x.float(), res.float(), acc.float()
    steps = 2 * k + C // 16
    _check(_conv(lib, BM, BN, xf, wp, bf, k, d, C, True), conv, mag, steps)
    _check(_conv(lib, BM, BN, xf, wp, bf, k, d, C, True, residual=rf), conv + res, mag + res.abs(), steps)
    _check(_conv(lib, BM, BN, xf, wp, bf, k, d, C, True, residual=rf, accum=af, div=3.0), (acc + conv + res) / 3,
           (acc.abs() + mag + res.abs()) / 3, steps)
    inplace = rf.clone()
    _check(_conv(lib, BM, BN, xf, wp, bf, k, d, C, True, residual=inplace, out=inplace), conv + res, mag + res.abs(),
           steps)


@pytest.mark.parametrize("BM,BN", INST)
@pytest.mark.parametrize("order", ["t_fast", "c_fast"])
def test_strided_conv_pre_input(lib, BM, BN, order):
    """conv_pre reads the mel through strides: channel-major [B, C, T] (unit stride along t: t_fast), or a token-major
    buffer of twice the channels read at every other channel (neither stride 1)"""
    B, C, N, T, k = 2, 32, 32, 2 * BM + 3, 7
    w, b = _rand(N, C, k, seed=11, scale=(C * k) ** -0.5), _rand(N, seed=12, scale=0.1)
    mel = _rand(B, C, T, seed=13)
    if order == "t_fast":
        buf = mel.float().contiguous()
        strides = (C * T, 1, T)
    else:
        wide = torch.full((B, T, 2 * C), float("nan"))
        wide[:, :, ::2] = mel.float().transpose(1, 2)
        buf = wide
        strides = (T * 2 * C, 2 * C, 2)
    ref = F.conv1d(mel, w, b, padding=3).transpose(1, 2)
    mag = F.conv1d(mel.abs(), w.abs(), b.abs(), padding=3).transpose(1, 2)
    out = _conv(lib, BM, BN, buf, hifigan.pack_conv(w.float()), b.float(), k, 1, N, False, strides=strides, T=T)
    _check(out, ref, mag, 2 * k + C // 16)


# (C_in, C_out, u, noise stride s) of the 44.1 kHz vocoder's five stages, the channels of the first three cut to
# 32 -> 16, 32 -> 16 and 64 -> 32 (the polyphase columns and the noise term depend on u, s and C_out's layout only)
STAGES = [(32, 16, 8, 64), (32, 16, 8, 8), (64, 32, 2, 4), (64, 32, 2, 2), (32, 16, 2, 1)]


@pytest.mark.parametrize("stage", range(5))
@pytest.mark.parametrize("T", [1, 2, 37])
def test_transposed_stage_with_source(lib, stage, T):
    """ConvTranspose1d(C_in, C_out, 2u, u, u / 2) in polyphase form + noise_convs(har_source), B 2, on every <BM, BN>"""
    Cin, Cout, u, s = STAGES[stage]
    nk, pad = (2 * s, s // 2) if stage < 4 else (1, 0)
    B = 2
    w, b = _rand(Cin, Cout, 2 * u, seed=stage, scale=Cin ** -0.5), _rand(Cout, seed=9, scale=0.1)
    wn, bn = _rand(Cout, 1, nk, seed=10, scale=nk ** -0.5), _rand(Cout, seed=11, scale=0.1)
    x, har = _rand(B, T, Cin, seed=12), torch.tanh(_rand(B, T * u * s, 1, seed=13)).float().double()
    xl = F.leaky_relu(x, 0.1)
    ref = (F.conv_transpose1d(xl.transpose(1, 2), w, b, stride=u, padding=u // 2) +
           F.conv1d(har.transpose(1, 2), wn, bn, stride=s, padding=pad)).transpose(1, 2)
    mag = (F.conv_transpose1d(xl.abs().transpose(1, 2), w.abs(), b.abs(), stride=u, padding=u // 2) +
           F.conv1d(har.abs().transpose(1, 2), wn.abs(), bn.abs(), stride=s, padding=pad)).transpose(1, 2)
    wp = hifigan.pack_conv(hifigan.polyphase(w.float(), u))
    xf, hf, bf = x.float(), har.float().reshape(B, -1).contiguous(), b.float()
    wnf, bnf = wn.float().reshape(Cout, nk).contiguous(), bn.float()
    for BM, BN in INST:
        out = torch.full((B, T * u, Cout), float("nan"))
        rc = lib.emu_hg_conv(BM, BN, _p(xf), T * Cin, Cin, 1, B, T, Cin, _p(wp), _p(bf), 3, 1, u * Cout, 1, None,
                             None, 1.0, u, _p(hf), _p(wnf), _p(bnf), nk, s, pad, _p(out))
        assert rc == 0
        # the noise term is an fp32 FMA chain of n_k taps after the conv: n_k more roundings of a sum bounded by mag
        _check(out, ref, mag, 6 + Cin // 16 + nk)


@pytest.mark.parametrize("T", range(1, 9))
def test_post(lib, T):
    """leaky_relu(x, 0.01) -> Conv1d(16 -> 1, k 7, padding 3) -> tanh, B 3 over a 2-CTA x 32-thread grid-stride loop.
    fp32 FMA over 7 16 = 112 terms: |err| <= 113 2^-24 mag before tanh, whose slope is at most 1, plus tanh's rounding"""
    B, C = 3, 16
    w, b = _rand(1, C, 7, seed=14, scale=0.1), _rand(1, seed=15, scale=0.1)
    x = _rand(B, T, C, seed=16)
    xl = F.leaky_relu(x.transpose(1, 2), 0.01)
    pre = F.conv1d(xl, w, b, padding=3)
    ref = torch.tanh(pre)
    mag = F.conv1d(xl.abs(), w.abs(), b.abs(), padding=3)
    out = torch.full((B, 1, T), float("nan"))
    xf, wf, bf = x.float().contiguous(), w.float()[0].t().contiguous(), b.float()      # alive across the call
    assert lib.emu_hg_post(_p(xf), _p(wf), _p(bf), B, T, C, 2, 32, _p(out)) == 0
    assert torch.isfinite(out).all()
    assert ((out.double() - ref).abs() <= 113 * 2.0 ** -24 * mag + 2.0 ** -23).all()


def test_kernels_under_address_sanitizer(tmp_path):
    """every input in a heap buffer of exactly its size, at T = 1 and the tile edges of each instantiation"""
    res = asan("emu_hifigan.cpp", tmp_path, "EMU_ASAN")
    assert res.returncode == 0 and "done 0" in res.stdout, res.stderr[-4000:]
