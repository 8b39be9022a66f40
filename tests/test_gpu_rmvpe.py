"""The RMVPE pitch extractor on the kernels (ddsp_svc_b200.E2E0 / RMVPE, csrc/rmvpe.cu) against float64: every launch
kind at each level's real shape, the GRU, the resampler and the log-mel, the whole network and RMVPE.infer_batch against
tests/rmvpe_oracle.py, the decode on constructed saliences, determinism and a warm call free of device syncs.  Measured
errors go to tests/report.py (B2D_PARITY_REPORT).

Bounds are relative RMS (and relative max) errors, 2.5 to 3 times the largest measured on an H100 80GB HBM3 at a 700 W
power limit (DESIGN.md section 4.17).  Decoded f0 is compared on the frames whose decision is robust: the top-1 / top-2
salience margin and |max - thred| both above 10 times the salience error bound.  There the voicing and argmax bin must
agree exactly and f0 is bounded; the other frames are counted and reported only."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import ops, rmvpe as R
from ddsp_svc_b200.hifigan import pack_conv
from tests import report
from tests import rmvpe_oracle as ro
from tests.golden import make_golden_rmvpe as mk

pytestmark = pytest.mark.gpu
DEV = "cuda"
# measured: one convolution <= 5.3e-7 RMS / 8.3e-7 max; the GRU <= 2.2e-7 absolute at T = 1024; the resampler
# <= 1.4e-6 relative max; the log-mel <= 3.9e-6 absolute; the whole seeded E2E0 <= 4.5e-5 RMS / 4.8e-4 max, growing
# with the frame count as the fp32 eager oracle's does (5.1e-4 / 1.6e-3 under cuDNN TF32 on the same case)
CONV_RMS, CONV_MAX = 1.5e-6, 2.5e-6
GRU_MAX = 6e-7
RESAMPLE_MAX = 4e-6
MEL_MAX = 1e-5
SAL_RMS, SAL_MAX = 1.2e-4, 1.5e-3      # salience, relative to its RMS / max (measured 4.5e-5 / 4.8e-4)
F0_REL = 1e-5


def _err(out, ref):
    out, ref = out.double().cpu(), ref.double().cpu()
    scale = ref.pow(2).mean().sqrt().item()
    return ((out - ref).pow(2).mean().sqrt().item() / scale, (out - ref).abs().max().item() / ref.abs().max().item())


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return scale * torch.randn(*shape, generator=g, dtype=torch.float64)


def _pack(w, b):
    return pack_conv(w.float().reshape(w.shape[0], w.shape[1], -1).to(DEV)), b.float().to(DEV)


def _nchw(x):
    return x.permute(0, 3, 1, 2)


# (B, T, F, C_in, C_out): the 3x3 convolutions of every level of E2E0(4, 1, (2, 2)) at T = 1024 frames (B = 1 also
# covers the deep levels' few tiles), plus a batch of 2
LEVELS = [(1, 64, 128, 16, 16), (1, 64, 64, 16, 32), (1, 32, 32, 64, 64), (2, 16, 16, 128, 128), (1, 64, 8, 256, 256),
          (1, 32, 4, 512, 512), (1, 32, 4, 256, 512),
          # level 0 of a 10 s clip (1024 frames: the 128-pixel, 16-column tiles) and level 1 of four of them (the
          # 128-pixel, 32-column tiles)
          (1, 1024, 128, 16, 16), (4, 512, 64, 32, 32)]


@pytest.mark.parametrize("B,T,Fq,Cin,Cout", LEVELS)
def test_conv3x3_relu_residual_slice(B, T, Fq, Cin, Cout):
    """relu(conv3x3 + bias) + residual, written into the second half of a wider (concat) buffer"""
    x, w, b = _rand(B, T, Fq, Cin, seed=1), _rand(Cout, Cin, 3, 3, seed=2, scale=(Cin * 9) ** -0.5), _rand(Cout, seed=3)
    res = _rand(B, T, Fq, Cout, seed=4)
    ref = F.relu(F.conv2d(_nchw(x), w, b, padding=1)) + _nchw(res)
    wp, bp = _pack(w, b)
    cat = torch.full((B, T, Fq, 2 * Cout), float("nan"), device=DEV)
    ops.rmvpe_conv(x.float().to(DEV), wp, bp, 3, Cout, act=1, residual=res.float().to(DEV), out=cat[..., Cout:])
    rel, mx = _err(_nchw(cat[..., Cout:]), ref)
    report.record("rmvpe/conv3x3/%dx%dx%d_%d_%d" % (B, T, Fq, Cin, Cout), rel_rms=rel, rel_max=mx)
    assert torch.isnan(cat[..., :Cout]).all()
    assert rel < CONV_RMS and mx < CONV_MAX, (rel, mx)


@pytest.mark.parametrize("B,T,Fq,Cin,Cout", [(1, 32, 128, 16, 32), (1, 16, 4, 256, 512), (2, 8, 16, 32, 64)])
def test_conv1x1_shortcut_from_slice(B, T, Fq, Cin, Cout):
    """the 1x1 shortcut with bias, read from a channel slice"""
    wide = _rand(B, T, Fq, 2 * Cin, seed=5)
    w, b = _rand(Cout, Cin, 1, 1, seed=6, scale=Cin ** -0.5), _rand(Cout, seed=7)
    ref = F.conv2d(_nchw(wide[..., Cin:]), w, b)
    wp, bp = _pack(w, b)
    out = ops.rmvpe_conv(wide.float().to(DEV)[..., Cin:], wp, bp, 1, Cout)
    rel, mx = _err(_nchw(out), ref)
    report.record("rmvpe/conv1x1/%dx%dx%d_%d_%d" % (B, T, Fq, Cin, Cout), rel_rms=rel, rel_max=mx)
    assert rel < CONV_RMS and mx < CONV_MAX, (rel, mx)


@pytest.mark.parametrize("B,T,Fq,Cin,Cout", [(1, 32, 4, 512, 256), (2, 8, 16, 64, 32), (1, 32, 64, 32, 16)])
def test_conv_transpose_polyphase(B, T, Fq, Cin, Cout):
    """ConvTranspose2d(3, stride 2, padding 1, output_padding 1) + bias + relu into the first half of the concat"""
    x = _rand(B, T, Fq, Cin, seed=8)
    wt, b = _rand(Cin, Cout, 3, 3, seed=9, scale=(Cin * 2.25) ** -0.5), _rand(Cout, seed=10)
    ref = F.relu(F.conv_transpose2d(_nchw(x), wt, b, stride=2, padding=1, output_padding=1))
    wp, bp = _pack(R.polyphase2d(wt), b)
    cat = torch.full((B, 2 * T, 2 * Fq, 2 * Cout), float("nan"), device=DEV)
    ops.rmvpe_conv(x.float().to(DEV), wp, bp, 2, 4 * Cout, act=1, up=True, out=cat[..., :Cout])
    rel, mx = _err(_nchw(cat[..., :Cout]), ref)
    report.record("rmvpe/convT/%dx%dx%d_%d_%d" % (B, T, Fq, Cin, Cout), rel_rms=rel, rel_max=mx)
    assert torch.isnan(cat[..., Cout:]).all()
    assert rel < CONV_RMS and mx < CONV_MAX, (rel, mx)


def test_first_conv_with_input_batchnorm():
    """C_in = 1: the input BatchNorm applies before the zero padding (not foldable into the bias at the edges)"""
    B, T = 2, 64
    mel = _rand(B, 128, T, seed=11) - 4
    w, b = _rand(16, 1, 3, 3, seed=12), _rand(16, seed=13)
    s, h = torch.tensor([0.7], dtype=torch.float64), torch.tensor([2.5], dtype=torch.float64)
    xin = mel.transpose(1, 2).unsqueeze(1) * s + h
    ref = F.relu(F.conv2d(xin, w, b, padding=1))
    x = mel.float().to(DEV).transpose(1, 2).unsqueeze(-1)
    out = ops.rmvpe_conv_small(x, w.float().to(DEV), b.float().to(DEV), relu=True, in_scale=s.float().to(DEV),
                               in_shift=h.float().to(DEV))
    rel, mx = _err(_nchw(out), ref)
    report.record("rmvpe/conv_cin1", rel_rms=rel, rel_max=mx)
    assert rel < CONV_RMS and mx < CONV_MAX, (rel, mx)


def test_cnn_head_layout():
    """cnn (16 -> 3, 3x3, bias) into the head's features, index c 128 + f"""
    B, T = 2, 32
    x, w, b = _rand(B, T, 128, 16, seed=14), _rand(3, 16, 3, 3, seed=15, scale=1 / 12), _rand(3, seed=16)
    ref = F.conv2d(_nchw(x), w, b, padding=1).transpose(1, 2).flatten(-2)
    out = ops.rmvpe_conv_small(x.float().to(DEV), w.float().to(DEV), b.float().to(DEV), head=True)
    rel, mx = _err(out, ref)
    report.record("rmvpe/cnn_head", rel_rms=rel, rel_max=mx)
    assert rel < CONV_RMS and mx < CONV_MAX, (rel, mx)


def test_pool_from_slice():
    x = _rand(2, 16, 32, 64, seed=17)
    out = ops.rmvpe_pool(x.float().to(DEV)[..., 32:])
    rel, mx = _err(_nchw(out), F.avg_pool2d(_nchw(x[..., 32:]), 2))
    assert mx < 1e-6, mx


@pytest.mark.parametrize("B", [1, 3, 6])
@pytest.mark.parametrize("T", [1, 32, 1024])
def test_gru(B, T):
    torch.manual_seed(0)
    g = torch.nn.GRU(384, 256, batch_first=True, bidirectional=True).double()   # fp32 weights, held exactly
    x = _rand(B, T, 384, seed=18)
    with torch.no_grad():
        ref = ro.gru(g, x)
        xg = torch.cat([F.linear(x, g.weight_ih_l0, g.bias_ih_l0), F.linear(x, g.weight_ih_l0_reverse,
                                                                            g.bias_ih_l0_reverse)], -1)
        whh = torch.stack([g.weight_hh_l0, g.weight_hh_l0_reverse]).float().to(DEV)
        bhh = torch.stack([g.bias_hh_l0, g.bias_hh_l0_reverse]).float().to(DEV)
    out = ops.rmvpe_gru(xg.float().to(DEV).contiguous(), whh.contiguous(), bhh.contiguous())
    err = (out.double().cpu() - ref).abs().max().item()
    report.record("rmvpe/gru/%dx%d" % (B, T), abs_max=err)
    assert err < GRU_MAX, err


@pytest.mark.parametrize("sr", [16000, 22050, 32000, 44100, 48000])
def test_resample(sr):
    n = 3 * sr // 2 + 37
    audio = _rand(2, n, seed=19, scale=0.3)
    ref = ro.resample(audio, sr)
    if sr == 16000:
        assert ref.shape[1] == n
        return
    table, width, orig, new = R.resample_table(sr)
    out = ops.rmvpe_resample(audio.float().to(DEV), table.to(DEV), new, orig, width, R.resampled_length(n, sr))
    assert out.shape == ref.shape
    err = (out.double().cpu() - ref).abs().max().item() / ref.abs().max().item()
    report.record("rmvpe/resample/%d" % sr, rel_max=err)
    assert err < RESAMPLE_MAX, err


@pytest.mark.parametrize("n", [513, 16000, 160 * 100 + 77])
def test_log_mel(n):
    audio = _rand(2, n, seed=20, scale=0.3)
    ref = ro.log_mel(audio)
    nf = ref.shape[-1]
    t_pad = 32 * ((nf - 1) // 32 + 1)
    basis = R.mel_basis()
    from ddsp_svc_b200.mel import _support
    out = ops.rmvpe_mel(audio.float().to(DEV), torch.hann_window(1024).to(DEV), torch.from_numpy(basis).to(DEV),
                        torch.from_numpy(_support(basis)).to(DEV), 160, t_pad)
    assert (out[:, nf:] == 0).all()
    err = (out[:, :nf].double().cpu().transpose(1, 2) - ref).abs().max().item()
    report.record("rmvpe/log_mel/%d" % n, abs_max=err)
    assert err < MEL_MAX, err


def _decode_checks(f0, sal, ref_f0, ref_sal, bound, name):
    """exact voicing and argmax on the robust frames, f0 relative error there; the other frames are reported"""
    ref_sal = ref_sal.double().cpu()
    top2 = ref_sal.topk(2, dim=-1).values
    robust = ((top2[..., 0] - top2[..., 1]) > 10 * bound) & ((top2[..., 0] - 0.03).abs() > 10 * bound)
    arg_ok = sal.double().cpu().argmax(-1) == ref_sal.argmax(-1)
    f0, ref_f0 = f0.double().cpu(), ref_f0.double().cpu()
    voiced_ok = (f0 > 0) == (ref_f0 > 0)
    assert bool(arg_ok[robust].all()) and bool(voiced_ok[robust].all())
    v = robust & (ref_f0 > 0)
    rel = ((f0 - ref_f0).abs() / ref_f0.clamp(min=1e-30))[v].max().item() if v.any() else 0.0
    differ = int(((f0 - ref_f0).abs() > F0_REL * ref_f0.abs())[~robust].sum())
    report.record(name, f0_rel_max=rel, robust=int(robust.sum()), other=int((~robust).sum()), other_differ=differ)
    assert rel < F0_REL, rel


@pytest.fixture(scope="module")
def full_model():
    with torch.no_grad():
        return ro.seeded_model().to(DEV)


@pytest.mark.parametrize("B,T", [(1, 32), (2, 64), (1, 96)])
def test_e2e0_whole(full_model, B, T):
    mel = _rand(B, 128, T, seed=21) - 4
    with torch.no_grad():
        ref = ro.salience(full_model, mel.to(DEV))
        m = full_model
        out = m(mel.float().to(DEV))
        again = m(mel.float().to(DEV))
        tf = ro.salience(m, mel.float().to(DEV), torch.float32)        # the reference's eager fp32 (cuDNN TF32)
    assert torch.equal(out, again)
    rel, mx = _err(out, ref)
    rel_tf, mx_tf = _err(tf, ref)
    report.record("rmvpe/e2e0/%dx%d" % (B, T), rel_rms=rel, rel_max=mx, eager_tf32_rel_rms=rel_tf,
                  eager_tf32_rel_max=mx_tf)
    assert rel < SAL_RMS and mx < SAL_MAX, (rel, mx)


def test_e2e0_reduced():
    with torch.no_grad():
        m = ro.seeded_model(n_blocks=1, en_de_layers=2, inter_layers=1)
        mel = _rand(2, 128, 300, seed=22) - 4
        m = m.to(DEV)
        ref = ro.salience(m, mel.to(DEV))
        out = m(mel.float().to(DEV))
    rel, mx = _err(out, ref)
    report.record("rmvpe/e2e0_reduced/2x300", rel_rms=rel, rel_max=mx)
    assert rel < SAL_RMS and mx < SAL_MAX, (rel, mx)


@pytest.mark.parametrize("sr,n", [(44100, 44100 + 123), (16000, 16000 * 2 + 5), (48000, 3 * 48000 // 2 + 7)])
def test_infer_batch(full_model, tmp_path, sr, n):
    path = tmp_path / "model.pt"
    torch.save({"model": full_model.state_dict()}, path)
    ex = R.RMVPE(str(path))
    t = torch.arange(n, dtype=torch.float64) / sr
    f = torch.tensor([[220.0], [330.0]], dtype=torch.float64)
    audio = 0.3 * torch.sin(2 * np.pi * f * t) + _rand(2, n, seed=23, scale=0.01)
    with torch.no_grad():
        ref_f0, ref_sal = ro.infer(full_model, audio.to(DEV), sr)
        f0 = ex.infer_batch(audio.float().to(DEV), sr)
        again = ex.infer_batch(audio.float().to(DEV), sr)
        sal, n_frames = ex.salience_batch(audio.float().to(DEV), sr)
        sal = sal[:, :n_frames]
    assert torch.equal(f0, again)
    assert f0.shape == ref_f0.shape
    rel, mx = _err(sal, ref_sal)
    report.record("rmvpe/infer_batch_salience/%d_%d" % (sr, n), rel_rms=rel, rel_max=mx)
    assert rel < SAL_RMS and mx < SAL_MAX, (rel, mx)
    _decode_checks(f0, sal, ref_f0, ref_sal, SAL_MAX * ref_sal.abs().max().item(), "rmvpe/infer_batch_f0/%d_%d" % (sr, n))
    one = ex.infer_from_audio(audio[0].numpy().astype(np.float32), sr)
    assert isinstance(one, np.ndarray) and one.shape == (ref_f0.shape[1],)
    assert np.array_equal(one, f0[0].cpu().numpy())


def test_decode_constructed():
    s = ro.constructed_saliences()
    ref = ro.decode(s[None])[0].double()             # fp32 like the reference's: 0.03f is not below thred there
    out = ops.rmvpe_decode(s[None].to(DEV).contiguous(), 12, 0.03)[0].double().cpu()
    assert torch.equal(out == 0, ref == 0)
    assert ((out - ref).abs() <= 2e-6 * ref.abs()).all(), (out, ref)


def test_determinism_and_sync_free(full_model, tmp_path):
    path = tmp_path / "model.pt"
    torch.save({"model": full_model.state_dict()}, path)
    ex = R.RMVPE(str(path))
    audio = _rand(2, 44100, seed=25, scale=0.3).float().to(DEV)
    first = ex.infer_batch(audio, 44100)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        second = ex.infer_batch(audio, 44100)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(first, second)


@pytest.mark.parametrize("name", list(mk.CASES))
def test_golden_replay(name, tmp_path):
    """the reference's recorded outputs through the kernels: the salience against its float64 run, and decoded f0
    under the robust-frame rule; audio cases through RMVPE.infer_from_audio"""
    d, m = mk.load(name)
    ref_sal = torch.from_numpy(d["hidden64"])
    with torch.no_grad():
        if "audio" in d:
            torch.save({"model": m.state_dict()}, tmp_path / "model.pt")
            ex = R.RMVPE(str(tmp_path / "model.pt"))
            f0_np = ex.infer_from_audio(d["audio"], int(d["sr"]))
            assert f0_np.shape == d["f0_32"][0].shape
            sal, n = ex.salience_batch(torch.from_numpy(d["audio"])[None].to(DEV), int(d["sr"]))
            sal, f0 = sal[:, :n], torch.from_numpy(f0_np)[None]
        else:
            mel = torch.from_numpy(d["mel"])
            n = mel.shape[-1]
            padded = torch.zeros(mel.shape[0], 128, 32 * ((n - 1) // 32 + 1))
            padded[..., :n] = mel
            sal = m.to(DEV)(padded.to(DEV))[:, :n]
            f0 = ops.rmvpe_decode(sal.contiguous(), n, 0.03)
    rel, mx = _err(sal, ref_sal)
    report.record("rmvpe/golden/%s" % name, rel_rms=rel, rel_max=mx)
    assert rel < SAL_RMS and mx < SAL_MAX, (rel, mx)
    _decode_checks(f0, sal, torch.from_numpy(d["f0_64"]), ref_sal, SAL_MAX * ref_sal.abs().max().item(),
                   "rmvpe/golden_f0/%s" % name)
