"""The diffusion cascade (ddsp_svc_b200/diffusion_vocoder.py) on the GPU: Unit2Mel's condition against a float64
restatement, the Unit2Mel / Unit2Wav / Unit2WavFast forwards with their draws passed in against the float64 sampler of
tests/diffusion_oracle.py for each of DDIM, PNDM, DPM-Solver, UniPC and DDPM, GaussianDiffusion's schedule cache (no
copy and no synchronisation after a warm call; a new k_step, speedup or method rebuilds it), and b2d_u2c_embed with a
phase, bit for bit against the formula it computed before its phase term became optional."""
import contextlib
import io
import json
import math

import pytest
import torch

from conversion_fixtures import HIFIGAN, write_synthetic_diff
from ddsp_svc_b200 import _lib
from ddsp_svc_b200 import diffusion_vocoder as dv
from ddsp_svc_b200.nsf_vocoder import Vocoder
from tests import diffusion_oracle, reflow_oracle, report, util
from tests.test_gpu_diffusion import SAMPLER_BOUND

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
METHODS = [("ddim", 10), ("pndm", 10), ("dpm-solver", 10), ("unipc", 10), (None, 1)]


def errors(got, truth):
    got, truth = got.double().cpu(), truth.double().cpu()
    return util.rms(got - truth) / util.rms(truth), float((got - truth).abs().max() / truth.abs().max())


def inputs(B, T, n_unit, seed):
    g = torch.Generator().manual_seed(seed)
    units = torch.randn(B, T, n_unit, generator=g)
    f0 = 110 + 300 * torch.rand(B, T, 1, generator=g)
    volume = 0.2 * torch.rand(B, T, 1, generator=g)
    return units.to(DEV), f0.to(DEV), volume.to(DEV)


def condition64(m, units, f0, volume, spk_id=None, spk_mix_dict=None, aug_shift=None):
    """diffusion/vocoder.py:206-215 in float64"""
    d = lambda t: t.detach().double()
    x = d(units) @ d(m.unit_embed.weight).t() + d(m.unit_embed.bias)
    x = x + (torch.log(1 + d(f0) / 700) @ d(m.f0_embed.weight).t() + d(m.f0_embed.bias))
    x = x + (d(volume) @ d(m.volume_embed.weight).t() + d(m.volume_embed.bias))
    if m.n_spk is not None and m.n_spk > 1:
        if spk_mix_dict is not None:
            for k, v in spk_mix_dict.items():
                x = x + v * d(m.spk_embed.weight)[int(k) - 1]
        else:
            x = x + d(m.spk_embed.weight)[spk_id.reshape(-1) - 1][:, None, :]
    if m.aug_shift_embed is not None and aug_shift is not None:
        x = x + (d(aug_shift).reshape(-1, 1, 1) / 5) * d(m.aug_shift_embed.weight)[:, 0]
    return x


@pytest.mark.parametrize("case", ["spk_id", "mix", "aug_b2"])
def test_unit2mel_condition_against_float64(case):
    torch.manual_seed(5)
    m = dv.Unit2Mel(768, 3, True, 128, 1, 64).to(DEV)
    B = 2 if case == "aug_b2" else 1
    units, f0, volume = inputs(B, 173, 768, 6)
    kw = dict(spk_id=torch.tensor([[2]] if B == 1 else [[1], [3]], device=DEV))
    if case == "mix":
        kw = dict(spk_mix_dict={1: 0.25, 3: 0.75})
    if case == "aug_b2":
        kw["aug_shift"] = torch.tensor([[3.0], [-2.0]], device=DEV)
    got = m.condition(units, f0, volume, **kw)
    want = condition64(m, units, f0, volume, **kw)
    rel = errors(got, want)[0]
    report.record("diffusion_cascade/condition/" + case, rel_rms=rel)
    assert got.shape == (B, 173, 256) and rel < 1e-5, rel


@pytest.fixture(scope="module")
def vocoder(tmp_path_factory):
    d = tmp_path_factory.mktemp("voc")
    with open(d / "config.json", "w") as f:
        json.dump(HIFIGAN, f)
    return Vocoder("nsf-hifigan", str(d / "model.ckpt"), device=DEV)      # extract only: the generator is not loaded


def build(kind):
    torch.manual_seed(11)
    if kind == "mel":
        m = dv.Unit2Mel(256, 2, True, 128, 2, 128)
        den, ref = m.decoder.denoise_fn, diffusion_oracle.WaveNet(128, 2, 128, 256)
    elif kind == "wav":
        m = dv.Unit2Wav(44100, 512, 256, 2, True, 128, 2, 128)
        den, ref = m.diff_model.denoise_fn, diffusion_oracle.WaveNet(128, 2, 128, 256)
    else:
        m = dv.Unit2WavFast(44100, 512, 2048, 256, 2, True, 128, 2, 128)
        den, ref = m.diff_model.denoise_fn, reflow_oracle.VelocityNet(128, 128, 128, 2)
    reflow_oracle.seeded_weights(den, 12, gain=0.5)
    ref.load_state_dict(den.state_dict(), strict=True)
    return m.to(DEV).eval(), ref.to(DEV, torch.float64).eval()


@pytest.mark.parametrize("method,speedup", METHODS)
@pytest.mark.parametrize("kind", ["mel", "wav", "fast"])
def test_forward_with_draws_against_float64(kind, method, speedup, vocoder):
    m, ref = build(kind)
    B, T, k_step = 1, 60, 40
    units, f0, volume = inputs(B, T, 256, 21)
    spk_id, aug = torch.tensor([[2]], device=DEV), torch.tensor([[1.5]], device=DEV)
    g = torch.Generator().manual_seed(22)
    noise = torch.randn(B, 1, 128, T, generator=g).to(DEV)
    steps = torch.randn(k_step, B, 1, 128, T, generator=g).to(DEV) if speedup == 1 else None
    ddsp_noise = (2 * torch.rand(B, T * 512, generator=g) - 1).to(DEV)
    with torch.no_grad():
        if kind == "mel":
            gt = (torch.linspace(-8.0, 0.5, 128)[None, None] + torch.randn(B, T, 128, generator=g)).to(DEV)
            got = m(units, f0, volume, spk_id=spk_id, aug_shift=aug, gt_spec=gt, infer_speedup=speedup, method=method,
                    k_step=k_step, noise=noise, step_noise=steps)
            cond = condition64(m, units, f0, volume, spk_id=spk_id, aug_shift=aug)
        else:
            if kind == "fast":
                ddsp_noise = torch.randn(B, T * 512, generator=g).to(DEV)
            got = m(units, f0, volume, spk_id=spk_id, aug_shift=aug, vocoder=vocoder, infer_speedup=speedup,
                    method=method, k_step=k_step, ddsp_noise=ddsp_noise, noise=noise, step_noise=steps)
            wav, hidden, _ = m.ddsp_model(units, f0, volume, spk_id=spk_id, aug_shift=aug, noise=ddsp_noise)
            gt = vocoder.extract(wav)
            cond = hidden if kind == "wav" else gt
        truth, _ = diffusion_oracle.sample(ref, cond, noise, gt, k_step, speedup, method, steps)
    rel, mx = errors(got, truth)
    report.record("diffusion_cascade/forward/%s/%s" % (kind, method), rel_rms=rel, rel_max=mx)
    assert got.shape == (B, T, 128)
    assert rel <= SAMPLER_BOUND["3xtf32"][0] and mx <= SAMPLER_BOUND["3xtf32"][1], (rel, mx)


def test_forward_draws_when_none_are_given(vocoder):
    m, _ = build("wav")
    units, f0, volume = inputs(1, 30, 256, 31)
    spk_id = torch.tensor([[1]], device=DEV)
    with torch.no_grad():
        torch.manual_seed(3)
        a = m(units, f0, volume, spk_id=spk_id, vocoder=vocoder, infer_speedup=5, method="ddim", k_step=20)
        torch.manual_seed(3)
        b = m(units, f0, volume, spk_id=spk_id, vocoder=vocoder, infer_speedup=5, method="ddim", k_step=20)
        c = m(units, f0, volume, spk_id=spk_id, vocoder=vocoder, infer_speedup=5, method="ddim", k_step=20)
    assert torch.equal(a, b) and not torch.equal(a, c)


def test_sampler_schedule_is_kept_after_a_warm_call():
    m, _ = build("mel")
    gd = m.decoder
    g = torch.Generator().manual_seed(41)
    cond = torch.randn(1, 50, 256, generator=g).to(DEV)
    gt = torch.randn(1, 50, 128, generator=g).to(DEV)
    noise = torch.randn(1, 1, 128, 50, generator=g).to(DEV)
    steps = torch.randn(30, 1, 1, 128, 50, generator=g).to(DEV)
    with torch.no_grad():
        for kw in (dict(method="dpm-solver", infer_speedup=5), dict(method="ddim", infer_speedup=10),
                   dict(method="ddim", infer_speedup=1, step_noise=steps)):
            first = gd(cond, gt_spec=gt, k_step=30, noise=noise, **kw)
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                again = gd(cond, gt_spec=gt, k_step=30, noise=noise, **kw)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            assert torch.equal(first, again), kw
        base = gd(cond, gt_spec=gt, k_step=30, noise=noise, method="ddim", infer_speedup=10)
        others = [gd(cond, gt_spec=gt, k_step=20, noise=noise, method="ddim", infer_speedup=10),
                  gd(cond, gt_spec=gt, k_step=30, noise=noise, method="ddim", infer_speedup=5),
                  gd(cond, gt_spec=gt, k_step=30, noise=noise, method="pndm", infer_speedup=10)]
        rebuilt = gd(cond, gt_spec=gt, k_step=30, noise=noise, method="ddim", infer_speedup=10)
        direct = gd._sample(cond, noise, gt, 30, 10, "ddim")
    assert torch.equal(base, rebuilt) and torch.equal(base, direct)
    assert not any(torch.equal(base, o) for o in others)


def _f32(x):
    return x.to(torch.float32)


def _fma(a, b, c):
    """fp32 fused multiply-add, as the kernel's FFMA computes it (the product is exact in float64)"""
    return _f32(a.double() * b.double() + c.double())


def test_u2c_embed_with_phase_is_unchanged():
    """x + (w_f0 lf + b_f0) + (w_ph ph + b_ph) + (w_vol vol + b_vol) + spk, then fma(w_aug, aug / 5, .): the kernel's
    fp32 operations before the phase became optional, restated with the same roundings"""
    B, T = 2, 300
    g = torch.Generator().manual_seed(51)
    x = torch.randn(B * T, 256, generator=g).to(DEV)
    f0 = (400 * torch.rand(B * T, generator=g)).to(DEV)
    phase = (6 * torch.rand(B * T, generator=g) - 3).to(DEV)
    vol = torch.rand(B * T, generator=g).to(DEV)
    emb = torch.randn(7, 256, generator=g).to(DEV)
    spk = torch.randn(B, 256, generator=g).to(DEV)
    aug = torch.tensor([2.0, -3.0], device=DEV)
    got = x.clone()
    _lib.check(_lib.lib().b2d_u2c_embed(got.data_ptr(), f0.data_ptr(), phase.data_ptr(), vol.data_ptr(),
                                        emb.data_ptr(), spk.data_ptr(), B, aug.data_ptr(), B, T, 0), "b2d_u2c_embed")
    lf = torch.log(1.0 + f0 / torch.full_like(f0, 700.0))[:, None]
    ph = (phase / torch.full_like(phase, float(torch.tensor(math.pi, dtype=torch.float32))))[:, None]
    a5 = (aug / torch.full_like(aug, 5.0)).repeat_interleave(T)[:, None]
    want = x + _fma(emb[0], lf, emb[1])
    want = want + _fma(emb[2], ph, emb[3])
    want = want + _fma(emb[4], vol[:, None], emb[5])
    want = want + spk.repeat_interleave(T, 0)
    want = _fma(emb[6], a5, want)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    # the null phase leaves the phase rows out
    nophase = x.clone()
    _lib.check(_lib.lib().b2d_u2c_embed(nophase.data_ptr(), f0.data_ptr(), 0, vol.data_ptr(), emb.data_ptr(), 0, 1,
                                        0, B, T, 0), "b2d_u2c_embed")
    want = x + _fma(emb[0], lf, emb[1])
    want = want + _fma(emb[4], vol[:, None], emb[5])
    torch.cuda.synchronize()
    assert torch.equal(nophase, want)


def test_load_model_vocoder_round_trip(tmp_path):
    with contextlib.redirect_stdout(io.StringIO()):
        _, path, _ = write_synthetic_diff(str(tmp_path), "DiffusionFast", n_chans=128, n_layers=2, encoder="hubertsoft")
        model, vocoder, args = dv.load_model_vocoder(path, device=DEV)
    assert isinstance(model, dv.Unit2WavFast) and args.model.type == "DiffusionFast" and vocoder.dimension == 128
