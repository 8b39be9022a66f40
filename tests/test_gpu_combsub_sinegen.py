"""GPU parity of the old CombSub synthesizer and of SineGen against the live-reference goldens
and the oracle, through the C ABI."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import CombSub, FixedControls, SineGen, SourceModuleHnNSF, ops, synthetic as syn
from tests import report, util
from tests.golden import cases as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P = G.SR, G.P
OFFICIAL_RMS = 1e-4
GATE_RMS = 2e-6


def _dev_ctrls(inp):
    return syn.split_views(inp["dense"].to(DEV), G.split_map(inp["case"]))


@pytest.mark.parametrize("name", [n for n, c in G.CASES.items() if c["kind"] == "combsub"])
def test_combsub_stages(name):
    inp = G.build_inputs(name)
    ref = util.port_outputs(name, inp)
    c = _dev_ctrls(inp)
    f0 = inp["f0"].to(DEV)
    fp, _ = ops.phase_scan(f0, P, SR)
    comb = ops.comb_source(f0, fp, P, SR).cpu()
    e_comb = util.rms(comb - ref["comb"])
    ir_h = ops.ir_build(c["harmonic_magnitude"], ops.IR_MAG_DYNAMIC, SR, f0_frames=f0).cpu()
    e_irh = (ir_h - ref["ir_harmonic"]).abs().max().item()
    # 1022-tap FIR on the oracle's intermediate signal ('auto' runs it on the FFT-domain kernel's 2048-point instance)
    y = ops.ltv_fir(ref["allpassed"].to(DEV), ref["ir_harmonic"].to(DEV).contiguous(), P).cpu()
    e_fir = util.rms(y - ref["harmonic"])
    report.record("combsub_stages/" + name, comb_rms=e_comb, comb_max=(comb - ref["comb"]).abs().max().item(),
                  ir_harmonic_max=e_irh, ir_harmonic_peak=ref["ir_harmonic"].abs().max().item(), fir1022_rms=e_fir,
                  harmonic_rms=util.rms(ref["harmonic"]))
    assert e_comb < 5e-6            # the reference's own fp32 comb sits ~1e-7 rms / 3e-6 max from exact math
    assert e_irh < 2e-6 * max(1.0, ref["ir_harmonic"].abs().max().item())
    assert e_fir < 1e-6


@pytest.mark.parametrize("name", [n for n, c in G.CASES.items() if c["kind"] == "combsub"])
def test_combsub_forward_matches_reference_golden(name):
    inp = G.build_inputs(name)
    gold = util.load_golden(name)
    case = inp["case"]
    B, nF = case["B"], case["nF"]
    hidden = torch.zeros(B, nF, 256, device=DEV)
    model = CombSub(SR, P, case["Ma"], case["Mh"], case["Mn"], unit2ctrl=FixedControls(_dev_ctrls(inp), hidden)).to(DEV)
    with torch.no_grad():
        signal, hid, (harm, nz) = model(None, inp["f0"].to(DEV), None, noise=inp["noise"].to(DEV))
    got = {"signal": signal.cpu().numpy(), "harmonic": harm.cpu().numpy(), "noise": nz.cpu().numpy()}
    errs = {k: util.rms(got[k] - gold[k]) for k in got}
    d = model.unit2ctrl.last_phase_frames.cpu().numpy() - gold["phase_frames"]
    d = (d + np.pi) % (2 * np.pi) - np.pi
    report.record("combsub_forward/" + name, signal_rms=util.rms(gold["signal"]), phase_frames_max=np.abs(d).max(),
                  **{k + "_err": v for k, v in errs.items()})
    assert np.abs(d).max() < 2e-6
    for k, e in errs.items():
        assert e < OFFICIAL_RMS and e < GATE_RMS, (k, e)
    assert torch.equal(signal, harm + nz)


def test_combsub_vs_float64_truth():
    name = "combsub_b2_f24"
    inp = G.build_inputs(name)
    truth = util.closed_form_outputs(name, inp)
    gold = util.load_golden(name)
    c = _dev_ctrls(inp)
    f0 = inp["f0"].to(DEV)
    fp, _ = ops.phase_scan(f0, P, SR)
    sig, _, _ = ops.combsub_synth(f0, fp, c["group_delay"], c["harmonic_magnitude"], c["noise_magnitude"], P, SR,
                                  noise_in=inp["noise"].to(DEV))
    e_gpu, e_ref = util.rms(sig.cpu().numpy() - truth["signal"]), util.rms(gold["signal"] - truth["signal"])
    report.record("combsub_truth", gpu_vs_truth=e_gpu, reference_vs_truth=e_ref)
    assert e_gpu < 1e-6


def test_combsub_full_size_config3b():
    """BASELINE config 3b shape (old CombSub, B=32 x 10 s, n_mag 256/512/256): finite, signal == harmonic + noise, the
    1022-tap FFT-domain FIR (2048-point instance) equals the one-thread-per-sample FIR on the same data, and two sampled
    utterances agree with the oracle port."""
    from oracle import torch_port as tp
    B, nF = 32, 861
    sm = syn.combsub_split_map(256, 512, 256)
    f0 = syn.make_f0(B, nF, SR, P)
    dense, ctrls = syn.make_ctrl(B, nF, sm)
    noise = syn.uniform_noise(B, nF * P, 21)
    dc = syn.split_views(dense.to(DEV), sm)
    f0d = f0.to(DEV)
    fp, _ = ops.phase_scan(f0d, P, SR)
    sig, harm, nz = ops.combsub_synth(f0d, fp, dc["group_delay"], dc["harmonic_magnitude"], dc["noise_magnitude"], P, SR,
                                      noise_in=noise.to(DEV))
    assert torch.isfinite(sig).all()
    assert torch.equal(sig, harm + nz)
    # the 2048-point FFT-domain instance at full size against the generic kernel (first 4 utterances: the generic
    # kernel is one thread per output sample x 1022 taps)
    comb = ops.comb_source(f0d, fp, P, SR)
    ir_h = ops.ir_build(dc["harmonic_magnitude"], ops.IR_MAG_DYNAMIC, SR, f0_frames=f0d)
    y_f = ops.ltv_fir(comb[:4], ir_h[:4], P)
    y_g = ops.ltv_fir(comb[:4], ir_h[:4], P, generic=True)
    e_fg = (y_f - y_g).abs().max().item()
    worst = 0.0
    for r in (3, 30):
        with torch.no_grad():
            ref = tp.combsub_forward(f0[r:r + 1], {k: v[r:r + 1] for k, v in ctrls.items()}, SR, P, noise=noise[r:r + 1])
        worst = max(worst, util.rms(sig[r:r + 1].cpu() - ref["signal"]))
    report.record("combsub_full", fft_vs_generic_max=e_fg, row_rms=worst, signal_rms=sig.pow(2).mean().sqrt().item())
    assert e_fg < 2e-6
    assert worst < GATE_RMS


@pytest.mark.parametrize("name", [n for n, c in G.CASES.items() if c["kind"] == "sinegen"])
def test_sinegen_matches_reference_golden(name):
    inp = G.build_inputs(name)
    gold = util.load_golden(name)
    case = inp["case"]
    gen = SineGen(SR, harmonic_num=case["harmonic_num"])
    out = gen(inp["f0"].to(DEV), case["upp"], rand_ini=inp["rand_ini"].to(DEV), noise=inp["noise"].to(DEV)).cpu().numpy()
    assert out.shape == gold["out"].shape
    e, m = util.rms(out - gold["out"]), np.abs(out - gold["out"]).max()
    report.record("sinegen/" + name, rms=e, max=m, ref_rms=util.rms(gold["out"]))
    assert e < OFFICIAL_RMS and e < GATE_RMS
    assert m < 2e-5


def test_sinegen_in_kernel_noise():
    """Throughput mode: Gaussian noise from Philox + Box-Muller inside the kernel."""
    B, nF, upp, dim = 3, 40, 512, 9
    gen = SineGen(SR, harmonic_num=dim - 1)
    f0 = torch.zeros(B, nF, device=DEV)          # all unvoiced: out = (sine_amp/3) * eps
    torch.manual_seed(5)
    a = gen(f0, upp)
    torch.manual_seed(5)
    b = gen(f0, upp)
    assert torch.equal(a, b)
    eps = (a / (0.1 / 3)).double().cpu().numpy()
    report.record("sinegen_noise", mean=eps.mean(), var=eps.var(), kurt=((eps - eps.mean()) ** 4).mean() / eps.var() ** 2)
    assert abs(eps.mean()) < 5e-3 and abs(eps.var() - 1) < 1e-2
    assert abs(((eps - eps.mean()) ** 4).mean() / eps.var() ** 2 - 3) < 0.05
    assert abs(np.corrcoef(eps[0, :, 0], eps[0, :, 1])[0, 1]) < 0.02
    assert abs(np.corrcoef(eps[0, :-1, 3], eps[0, 1:, 3])[0, 1]) < 0.02
    # voiced part: deterministic sines + small noise; shard invariance of the noise stream
    f0v = syn.make_f0(B, nF, SR, upp)[..., 0].to(DEV)
    ri = torch.zeros(dim)
    x = ops.sinegen(f0v, upp, SR, dim, ri, seed=9)
    y = ops.sinegen(f0v[1:], upp, SR, dim, ri, seed=9, utterance_offset=1)
    assert torch.equal(x[1:], y)


def test_sinegen_full_size_config5():
    """BASELINE config 5 shape: B=64 x 10 s x 9 harmonics (1 GB output)."""
    B, nF, upp, dim = 64, 861, 512, 9
    f0 = syn.make_f0(B, nF, SR, upp, unvoiced_fraction=0.1)[..., 0]
    ri = torch.rand(dim); ri[0] = 0
    out = ops.sinegen(f0.to(DEV), upp, SR, dim, ri, seed=3)
    assert out.shape == (B, nF * upp, dim) and torch.isfinite(out).all()
    # one utterance against the oracle with its noise removed: feed zeros as noise
    from oracle import torch_port as tp
    row = 11
    z = torch.zeros(1, nF * upp, dim)
    ref = tp.sinegen_forward(f0[row:row + 1], upp, SR, dim - 1, rand_ini=ri.reshape(1, 1, -1), noise=z)["out"]
    got = ops.sinegen(f0[row:row + 1].to(DEV), upp, SR, dim, ri, noise_in=z.to(DEV)).cpu()
    e = util.rms(got - ref)
    report.record("sinegen_full", row_rms=e, row_max=(got - ref).abs().max().item())
    assert e < GATE_RMS


# ---- SourceModuleHnNSF: SineGen + tanh(Linear(9 -> 1)) in one kernel (nsf_hifigan/models.py:168-204) ----
@pytest.mark.parametrize("name", [n for n, c in G.CASES.items() if c["kind"] == "source_module"])
def test_source_module_matches_reference_golden(name):
    inp = G.build_inputs(name)
    gold = util.load_golden(name)
    case = inp["case"]
    m = SourceModuleHnNSF(SR, harmonic_num=case["harmonic_num"])
    m.load_state_dict({"l_linear.weight": torch.from_numpy(gold["weight"]), "l_linear.bias": torch.from_numpy(gold["bias"])})
    m = m.to(DEV).eval()
    with torch.no_grad():
        out = m(inp["f0"].to(DEV), case["upp"], rand_ini=inp["rand_ini"].to(DEV), noise=inp["noise"].to(DEV)).cpu().numpy()
    assert out.shape == gold["out"].shape == (case["B"], case["nF"] * case["upp"], 1)
    e, mx = util.rms(out - gold["out"]), np.abs(out - gold["out"]).max()
    report.record("source_module/" + name, rms=e, max=mx, ref_rms=util.rms(gold["out"]))
    assert e < OFFICIAL_RMS and e < GATE_RMS
    assert mx < 2e-5


def test_source_module_equals_linear_tanh_of_sinegen():
    """the fused kernel against tanh(linear(.)) applied to the UNFUSED kernel's own output, in-kernel noise on:
    same Philox stream in both, so the two agree to fp32 rounding of a 9-term dot product."""
    B, nF, upp, dim = 3, 40, 512, 9
    f0v = syn.make_f0(B, nF, SR, upp, seed=21, unvoiced_fraction=0.2)[..., 0].contiguous().to(DEV)
    ri = torch.rand(dim); ri[0] = 0
    g = torch.Generator().manual_seed(3)
    w, b = torch.randn(1, dim, generator=g), 0.37
    sines = ops.sinegen(f0v, upp, SR, dim, ri, seed=77, utterance_offset=5)
    want = torch.tanh(torch.nn.functional.linear(sines.double(), w.double().to(DEV)) + b)
    got = ops.source_module(f0v, upp, SR, dim, ri, w, b, seed=77, utterance_offset=5)
    assert got.shape == (B, nF * upp, 1)
    err = (got.double() - want).abs().max().item()
    report.record("source_module_fused_vs_unfused", max=err)
    assert err < 2e-6


@pytest.mark.parametrize("impl", ["v1", "v2", "v2p"])
@pytest.mark.parametrize("upp,nF", [(130, 5), (512, 7), (3, 9)])
def test_sinegen_kernel_variants_match_oracle(impl, upp, nF):
    """every kernel variant (one / four samples per thread, scalar / packed f32x2) against the oracle port on
    explicit noise, including hop sizes that are not powers of two and T not a multiple of 4 (ragged last thread)."""
    from oracle import torch_port as tp
    B, dim = 2, 9
    f0 = syn.make_f0(B, nF, SR, upp, seed=31, unvoiced_fraction=0.3)[..., 0].contiguous()
    g = torch.Generator().manual_seed(8)
    ri = torch.rand(dim, generator=g); ri[0] = 0
    z = torch.randn(B, nF * upp, dim, generator=g)
    w, bias = torch.randn(1, dim, generator=g) / 3, torch.tensor([0.1])
    ref = tp.source_module_forward(f0, upp, SR, w, bias, dim - 1, rand_ini=ri.reshape(1, 1, -1), noise=z)
    ops.set_sinegen_impl(impl)
    try:
        got = ops.sinegen(f0.to(DEV), upp, SR, dim, ri, noise_in=z.to(DEV)).cpu()
        merged = ops.source_module(f0.to(DEV), upp, SR, dim, ri, w, float(bias), noise_in=z.to(DEV)).cpu()
        # in-kernel noise: fused and unfused draw the same stream inside one variant
        a = ops.sinegen(f0.to(DEV), upp, SR, dim, ri, seed=5)
        bm = ops.source_module(f0.to(DEV), upp, SR, dim, ri, w, float(bias), seed=5)
        want = torch.tanh(torch.nn.functional.linear(a.double(), w.double().to(DEV)) + float(bias))
    finally:
        ops.set_sinegen_impl("auto")
    e_sines = (got - ref["sines"]).abs().max().item()
    e_merged = (merged - ref["out"]).abs().max().item()
    report.record("sinegen_variant/%s/upp%d" % (impl, upp), max=e_sines, fused_max=e_merged)
    assert got.shape == ref["sines"].shape and merged.shape == ref["out"].shape
    assert e_sines < 2e-5 and util.rms((got - ref["sines"]).numpy()) < 1e-6
    assert e_merged < 2e-5
    assert (bm.double() - want).abs().max().item() < 2e-6


def test_sinegen_philox7_noise_statistics():
    """`v2r7` draws its normals from Philox4x32-7 (the smallest round count reported to pass BigCrush) instead of -10.
    Checked here on 2.4 M samples: Kolmogorov-Smirnov distance to N(0, 1), autocorrelation at lags 1..16 along time, correlation
    between harmonics, between utterances, between different seeds and with the 10-round stream of the same counters."""
    B, nF, upp, dim = 8, 64, 512, 9
    f0 = torch.zeros(B, nF, device=DEV)
    ri = torch.zeros(dim)
    draw = lambda impl, seed: (ops.sinegen(f0, upp, SR, dim, ri, seed=seed) / (0.1 / 3)).double().cpu()
    try:
        ops.set_sinegen_impl("v2r7")
        a, a2 = draw("v2r7", 21), draw("v2r7", 22)
        assert torch.equal(a, draw("v2r7", 21))                         # deterministic per seed
        ops.set_sinegen_impl("v2")
        ten = draw("v2", 21)
    finally:
        ops.set_sinegen_impl("auto")
    x = a.reshape(-1)
    n = x.numel()
    xs, _ = torch.sort(x)
    cdf = 0.5 * (1 + torch.erf(xs / 2 ** 0.5))
    i = torch.arange(1, n + 1, dtype=torch.float64)
    ks = torch.max(torch.max(i / n - cdf), torch.max(cdf - (i - 1) / n)).item()
    t = a[:, :, 0]                                                       # harmonic 0 along time, per utterance
    t = t - t.mean(dim=1, keepdim=True)
    lags = [float((t[:, :-k] * t[:, k:]).mean() / t.var()) for k in range(1, 17)]
    flat = a.reshape(-1, dim)
    cross_h = (torch.corrcoef(flat.T) - torch.eye(dim)).abs().max().item()
    cross_u = abs(torch.corrcoef(torch.stack([a[0].reshape(-1), a[1].reshape(-1)]))[0, 1].item())
    cross_seed = abs(torch.corrcoef(torch.stack([x, a2.reshape(-1)]))[0, 1].item())
    cross_rounds = abs(torch.corrcoef(torch.stack([x, ten.reshape(-1)]))[0, 1].item())
    report.record("sinegen_noise/v2r7_ks", n=n, ks=ks, ks_bound=1.63 / n ** 0.5, max_lag_corr=max(abs(v) for v in lags), cross_harmonic=cross_h,
                  cross_utterance=cross_u, cross_seed=cross_seed, cross_rounds=cross_rounds, mean=x.mean().item(), var=x.var().item())
    assert ks < 1.63 / n ** 0.5                                          # 1 % critical value of the KS test
    tol = 4.5 / (n / dim) ** 0.5                                         # ~4.5 sigma of a sample correlation
    assert max(abs(v) for v in lags) < 4.5 / (t.numel()) ** 0.5 * 1.5 and cross_h < tol * 1.5
    assert cross_u < 4.5 / (n / B) ** 0.5 and cross_seed < 4.5 / n ** 0.5 and cross_rounds < 4.5 / n ** 0.5


@pytest.mark.parametrize("impl", ["v1", "v2p", "v2r7"])
def test_sinegen_in_kernel_noise_moments_per_variant(impl):
    B, nF, upp, dim = 4, 64, 512, 9
    f0 = torch.zeros(B, nF, device=DEV)            # unvoiced: out = (sine_amp/3) * eps, so eps is observable
    ri = torch.zeros(dim)
    ops.set_sinegen_impl(impl)
    try:
        eps = (ops.sinegen(f0, upp, SR, dim, ri, seed=11) / (0.1 / 3)).double().cpu()
    finally:
        ops.set_sinegen_impl("auto")
    n = eps.numel()
    mean, var = eps.mean().item(), eps.var().item()
    kurt = ((eps - mean) ** 4).mean().item() / var ** 2
    assert abs(mean) < 5 / n ** 0.5 and abs(var - 1) < 0.01 and abs(kurt - 3) < 0.03
    # no correlation between harmonics or between neighbouring samples
    flat = eps.reshape(-1, dim)
    c = torch.corrcoef(flat.T)
    assert (c - torch.eye(dim)).abs().max().item() < 0.01
    assert abs(torch.corrcoef(torch.stack([flat[:-1, 0], flat[1:, 0]]))[0, 1].item()) < 0.01
    assert eps.abs().max().item() > 4.0            # tails present (24-bit radius)
    report.record("sinegen_noise/" + impl, mean=mean, var=var, kurt=kurt)
