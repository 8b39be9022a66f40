"""csrc/rmvpe.cu's kernels without a GPU: their source executed on the CPU (tests/emu/host_emu.h, with its warp,
mma.sync, cp.async and cluster models) against float64 torch, then under AddressSanitizer.  rv_conv runs every <BM, BN>
instantiation at both tile shapes (tF = F < BM / 4 and tF = BM / 4) with its weights packed by the package's own
packers (hifigan.pack_conv, rmvpe.polyphase2d); rv_gru runs as 8-CTA clusters over full, partial and several batch
groups.  The kernels run on hardware in tests/test_gpu_rmvpe.py.

rv_conv's bound per output element is test_emu_hifigan.py's: 3xTF32 leaves each product within 3 2^-22 of exact, and
the fp32 sums of the 2 k^2 mma results per 16-channel chunk, the per-chunk adds, the bias and the residual each round
within 2^-24 of a partial sum bounded by `mag` (the convolution of |x| and |w| plus |bias| and |residual|).  ReLU and
the sigmoid have slopes <= 1; expf adds a few ulp of the output.  Integer decisions (rv_decode's voicing) are exact."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from ddsp_svc_b200 import hifigan, rmvpe
from tests import rmvpe_oracle as ro
from tests.emu_harness import asan, shared

INST = [(64, 32), (64, 16), (128, 32), (128, 16)]
NAN = float("nan")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return shared("emu_rmvpe.cpp", tmp_path_factory)


def _rand(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(*shape, generator=g, dtype=torch.float64)).float().double()


def _p(t):
    return None if t is None else t.data_ptr()


def _bound(mag, steps, ref):
    return (3 * 2.0 ** -22 + (steps + 3) * 2.0 ** -24) * mag + 2.0 ** -21 * ref.abs()


@pytest.mark.parametrize("BM,BN", INST)
@pytest.mark.parametrize("tile", ["tF_is_F", "tF_is_BM_over_4"])
@pytest.mark.parametrize("kind", ["k1", "k3", "up"])
def test_conv(lib, BM, BN, tile, kind):
    """[B, T, F, C] slices of wider buffers (ldx > Cin, ldo > N with NaN siblings that must stay NaN), T not a multiple
    of tT, n_valid < N for k 3; act 0 / 1 / 2 and the residual rotate over the cases"""
    k = {"k1": 1, "k3": 3, "up": 2}[kind]
    F_ = 4 if tile == "tF_is_F" else BM // 4
    tT = BM // min(F_, BM // 4)
    B, T, Cin, N = 2, tT + 3, 48, 32                                  # 3 chunks: both stages refilled
    case = INST.index((BM, BN)) + 4 * ["k1", "k3", "up"].index(kind)
    act, with_res = case % 3, case % 2 == 0 and kind != "up"
    n_valid = N - 6 if kind == "k3" else N
    ldx, ldo = Cin + 16, N + 8
    x = _rand(B, T, F_, Cin, seed=case)
    xbuf = torch.full((B, T, F_, ldx), NAN)
    xbuf[..., :Cin] = x.float()
    xin = x.permute(0, 3, 1, 2)                                        # [B, Cin, T, F]
    if kind == "up":
        Cout = N // 4
        wt, b = _rand(Cin, Cout, 3, 3, seed=40 + case, scale=(9 * Cin) ** -0.5), _rand(Cout, seed=41, scale=0.1)
        conv = lambda a, w_, b_: F.conv_transpose2d(a, w_, b_, stride=2, padding=1, output_padding=1)
        ref, mag = conv(xin, wt, b), conv(xin.abs(), wt.abs(), b.abs())
        w4 = rmvpe.polyphase2d(wt.float())                             # [4 Cout, Cin, 2, 2]
        wp = hifigan.pack_conv(w4.reshape(N, Cin, 4).contiguous())
        out = torch.full((B, 2 * T, 2 * F_, ldo), NAN)
        res = None
    else:
        w, b = _rand(N, Cin, k, k, seed=40 + case, scale=(k * k * Cin) ** -0.5), _rand(N, seed=41, scale=0.1)
        ref = F.conv2d(xin, w, b, padding=k // 2)
        mag = F.conv2d(xin.abs(), w.abs(), b.abs(), padding=k // 2)
        wp = hifigan.pack_conv(w.float().reshape(N, Cin, k * k).contiguous())
        out = torch.full((B, T, F_, ldo), NAN)
        res = _rand(B, T, F_, N, seed=50 + case) if with_res else None
    ref, mag = ref.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)
    if act == 1:
        ref = ref.clamp_min(0)
    elif act == 2:
        ref = torch.sigmoid(ref)
    if res is not None:
        ref, mag = ref + res, mag + res.abs()
    resf, bf = (res.float().contiguous() if res is not None else None), b.float()
    rc = lib.emu_rv_conv(BM, BN, _p(xbuf), ldx, B, T, F_, Cin, _p(wp), _p(bf), k, N, n_valid, act, int(kind == "up"),
                         _p(resf), N, _p(out), ldo)
    assert rc == 0
    Nout = N // 4 if kind == "up" else n_valid
    got = out[..., :Nout].double()
    assert torch.isnan(out[..., Nout:]).all(), "a column past n_valid or a sibling slice was written"
    assert torch.isfinite(got).all(), "unwritten or poisoned elements"
    ref, mag = ref[..., :Nout], mag[..., :Nout]
    err = (got - ref).abs()
    assert (err <= _bound(mag, 2 * k * k + Cin // 16, ref)).all(), err.max().item()
    assert ((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item() < 1e-6


@pytest.mark.parametrize("mode", ["input_batchnorm", "head"])
def test_conv_small(lib, mode):
    """the first convolution (C_in 1, the input BatchNorm on real pixels before the zero padding) and `cnn` (C_out 3,
    head layout c F + f).  fp32 FMA over 9 C_in terms: |err| <= (9 C_in + 2) 2^-24 mag"""
    B, T, F_ = 2, 5, 6
    if mode == "head":
        Cin, Cout = 16, 3
        x = _rand(B, T, F_, Cin, seed=1)
        scale = shift = None
        xin = x.permute(0, 3, 1, 2)
    else:
        Cin, Cout = 1, 16
        x = _rand(B, T, F_, 1, seed=1)
        scale, shift = _rand(1, seed=2), _rand(1, seed=3)
        xin = (x * scale + shift).permute(0, 3, 1, 2)
    w, b = _rand(Cout, Cin, 3, 3, seed=4, scale=(9 * Cin) ** -0.5), _rand(Cout, seed=5, scale=0.1)
    ref, mag = F.conv2d(xin, w, b, padding=1), F.conv2d(xin.abs(), w.abs(), b.abs(), padding=1)
    if mode == "head":
        ref, mag = ref.permute(0, 2, 1, 3), mag.permute(0, 2, 1, 3)          # [B, T, Cout, F]
        out = torch.full((B, T, Cout, F_), NAN)
    else:
        ref, mag = ref.clamp_min(0).permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)
        out = torch.full((B, T, F_, Cout), NAN)
    xf, wf, bf = x.float().contiguous(), w.float().contiguous(), b.float()
    sf, hf = (scale.float(), shift.float()) if scale is not None else (None, None)
    rc = lib.emu_rv_conv_small(_p(xf), T * F_ * Cin, F_ * Cin, Cin, 1, B, T, F_, Cin, _p(sf), _p(hf), _p(wf), _p(bf), 3,
                               Cout, int(mode != "head"), int(mode == "head"), _p(out), Cout)
    assert rc == 0 and torch.isfinite(out).all()
    assert ((out.double() - ref).abs() <= (9 * Cin + 4) * 2.0 ** -24 * (mag + ref.abs())).all()


def test_pool(lib):
    """AvgPool2d(2) of a channel slice (ldx > C): four fp32 adds and an exact * 0.25"""
    B, T, F_, C, ldx = 2, 6, 8, 16, 24
    x = _rand(B, T, F_, ldx, seed=7)
    ref = F.avg_pool2d(x[..., :C].permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    mag = F.avg_pool2d(x[..., :C].abs().permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    xf, out = x.float().contiguous(), torch.full((B, T // 2, F_ // 2, C), NAN)
    assert lib.emu_rv_pool(_p(xf), ldx, B, T, F_, C, _p(out)) == 0
    assert ((out.double() - ref).abs() <= 3 * 2.0 ** -24 * mag).all()


@pytest.mark.parametrize("B,T", [(1, 1), (3, 2), (4, 2), (5, 2), (9, 1), (1, 17)])
def test_gru(lib, B, T):
    """8-CTA clusters per direction: one full group (B 4), partial groups (1, 3), a full and a partial one (5), three
    groups (9), and 17 steps of h through distributed shared memory.  Against tests/rmvpe_oracle.gru in float64 with
    the kernel's fp32 input projection as xg.  fp32: 256-term FMA dots of |w| <= 1/16 against |h| < 1 and fp32 gates;
    the recurrence is contractive at these weights, so the bound does not grow with T"""
    torch.manual_seed(0)
    g = nn.GRU(384, 256, batch_first=True, bidirectional=True).double()
    with torch.no_grad():
        for p in g.parameters():
            p.copy_(p.float().double())
    x = _rand(B, T, 384, seed=B * 100 + T)
    xg = torch.cat([F.linear(x, g.weight_ih_l0, g.bias_ih_l0), F.linear(x, g.weight_ih_l0_reverse,
                                                                         g.bias_ih_l0_reverse)], -1).float()
    ref = ro.gru(g, x)
    whh = torch.stack([g.weight_hh_l0, g.weight_hh_l0_reverse]).float().contiguous()
    bhh = torch.stack([g.bias_hh_l0, g.bias_hh_l0_reverse]).float().contiguous()
    out = torch.full((B, T, 512), NAN)
    assert lib.emu_rv_gru(_p(xg), _p(whh), _p(bhh), B, T, _p(out)) == 0
    assert torch.isfinite(out).all()
    assert (out.double() - ref).abs().max().item() < 2e-6


def test_decode_constructed_saliences(lib):
    """rmvpe_oracle.constructed_saliences (ties, edges, sub-threshold peaks) as 2 utterances of 6 frames in a t_pad 8
    buffer whose padding rows are NaN: the voicing decision matches the reference's fp32 decode exactly (0.03f is not
    below thred there), f0 to the fp32 rounding of a 9-term weighted mean and exp2f"""
    sal = ro.constructed_saliences().float()
    want = ro.decode(sal[None])[0].double().reshape(2, 6)
    buf = torch.full((2, 8, 360), NAN)
    buf[:, :6] = sal.float().reshape(2, 6, 360)
    f0 = torch.full((2, 6), NAN)
    assert lib.emu_rv_decode(_p(buf), 2, 8, 6, 0.03, _p(f0)) == 0
    assert torch.equal(f0 == 0, want == 0)
    assert ((f0.double() - want).abs() <= 2e-6 * want.abs()).all()


def test_kernels_under_address_sanitizer(tmp_path):
    """every input in a heap buffer of exactly its size: rv_conv at both tile shapes, k 1 / 3 / up with n_valid < N,
    rv_conv_small in both modes, rv_pool, rv_gru with a partial batch group, rv_resample, rv_mel at n 513 and 1101 and
    rv_decode with padding rows"""
    res = asan("emu_rmvpe.cpp", tmp_path, "EMU_ASAN")
    assert res.returncode == 0 and "done 0" in res.stdout, res.stderr[-4000:]


def _resample_mag(audio, sr):
    """rmvpe_oracle.resample's convolution with |table| over |audio|: the magnitude sum of each output's terms"""
    table, width, orig, new = rmvpe.resample_table(sr)
    return ro.resample(audio.abs(), sr, tabs=dict(resample=(table.double().abs(), width, orig, new)))


@pytest.mark.parametrize("sr", [22050, 48000])
def test_resample(lib, sr):
    """torchaudio's Resample(sr, 16000, lowpass_filter_width 128) as a polyphase FIR over a 3-CTA grid-stride loop, B 2,
    both utterance edges inside the taps.  One fp32 FMA chain of `taps` terms: |err| <= taps 2^-24 mag"""
    B, n = 2, sr // 20 + 37
    audio = _rand(B, n, seed=sr, scale=0.3)
    ref, mag = ro.resample(audio, sr), _resample_mag(audio, sr)
    table, width, orig, new = rmvpe.resample_table(sr)
    n_out = rmvpe.resampled_length(n, sr)
    out = torch.full((B, n_out), NAN)
    xf = audio.float().contiguous()
    assert lib.emu_rv_resample(_p(xf), B, n, _p(table), new, orig, table.shape[1], width, n_out, _p(out)) == 0
    assert out.shape == ref.shape and torch.isfinite(out).all()
    assert ((out.double() - ref).abs() <= table.shape[1] * 2.0 ** -24 * mag).all()


@pytest.mark.parametrize("n", [513, 1024 + 77])
def test_log_mel(lib, n):
    """spec.py's log-mel (center, reflect) through fft_smem.cuh's shared-memory FFT, two frames per transform, an odd
    frame count, B 2 and t_pad 32, whose padding frames must be exactly zero.  Bound: a radix FFT of 1024 points in
    fp32 (with fp32 twiddles) keeps each bin within 4 (log2 1024 + 2) 2^-24 of the frame's sum |w x|; the filter sums
    then move each mel value by at most that times the filter's weight sum, a relative change of the log's argument
    (clamped at 1e-5)"""
    from ddsp_svc_b200.mel import _support
    B, hop, t_pad = 2, 160, 32
    audio = _rand(B, n, seed=n, scale=0.3)
    ref = ro.log_mel(audio).transpose(1, 2)                            # [B, nf, 128]
    nf = ref.shape[1]
    basis = rmvpe.mel_basis()
    window = torch.hann_window(1024, dtype=torch.float32)
    frames = F.pad(audio[:, None], (512, 512), mode="reflect")[:, 0].unfold(-1, 1024, hop)[:, :nf]
    S = (frames.abs() * window.double()).sum(-1, keepdim=True)        # [B, nf, 1]
    wsum = torch.from_numpy(basis).double().sum(-1)                    # [128]
    mel = ref.exp()
    bound = 4 * (10 + 2) * 2.0 ** -24 * S * wsum / mel.clamp_min(1e-5) + 4 * 2.0 ** -24 * ref.abs()
    out = torch.full((B, t_pad, 128), NAN)
    af, bf, lohi = audio.float().contiguous(), torch.from_numpy(basis), torch.from_numpy(_support(basis))
    assert lib.emu_rv_mel(_p(af), B, n, _p(window), _p(bf), _p(lohi), hop, 1 + n // hop, t_pad, _p(out)) == 0
    assert 1 + n // hop == nf and torch.equal(out[:, nf:], torch.zeros(B, t_pad - nf, 128))
    err = (out[:, :nf].double() - ref).abs()
    assert (err <= bound).all(), (err - bound).max().item()
