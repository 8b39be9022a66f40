"""GPU: every synthesizer, its stage kernels and its selectable variants at the input regimes of tests/regimes.py --
the pitches a tracker returns and the control values a trained network emits -- not only at synthetic.py's benchmark
distribution.  The CPU emulator evaluates the SFU intrinsics exactly, so the range reduction of __sincosf, the error
of __expf at large arguments and tanh's saturation are only visible here.

Pairing (the same for Sins, CombSub, CombSubFast, CombSubSuperFast; SineGen / source_module take the pitch column):

    pitch \\ control   trained  phase_turns  saturated_gd  hot  cold  mixed_rows
    low                  x                      x
    high                           x                             x
    octave_jumps                                x           x
    onsets               x                                               x
    glide                          x                        x
    near_zero                                                    x       x

Pass criterion.  A fixed absolute gate cannot hold here: at 800 rad of all-pass phase, or with the training phase's
fp32 cumsum, the reference's own fp32 arithmetic is tens to hundreds of ppm from exact.  Each case computes the float64
closed form (truth), the reference's arithmetic in fp32 on the CPU (ref32, oracle.torch_port: what the kernels promise
to match) and the GPU result, and asserts per utterance row

    rms(gpu - truth) <= max(floor, RMS_FACTOR x rms(ref32 - truth)),   floor = 2e-6 x max(1, rms(truth) / 0.01)
    max|gpu - truth| <= max(8 x floor, MAX_FACTOR x max|ref32 - truth|)

plus finite outputs and signal == harmonic + noise.  Per row, so that in mixed_rows a read across the row boundary
shows as an error of 1e10 floors in the cold row.  The three errors of every case go to tests.report.
"""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import ops, synthetic as syn
from oracle import closed_form as cf
from oracle import torch_port as tp
from tests import regimes as R
from tests import report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P, WIN = R.SR, R.P, R.WIN
# Calibrated on an H100 80GB HBM3 (700 W): wherever ref32's error is above the floor the kernels' error equals it to
# within 2 % in RMS (worst 1.02, CombSub training phase at glide-phase_turns) and 3 % in max-abs, because both round the
# same phase to fp32 -- the factors leave a kernel room for its own error of the size of the reference's, no more
RMS_FACTOR, MAX_FACTOR = 2.0, 3.0
# the entries whose fp32 reference is furthest from float64 (tests/test_regimes_oracle.py), plus the Nyquist-floor one
STAGE_CASES = [("octave_jumps", "saturated_gd"), ("onsets", "trained"), ("high", "phase_turns")]
MODES = [(s, i) for s in R.SPLITS for i in ((True, False) if s in R.HAS_INFER else (True,))]


def gpu_forward(inp, infer=True):
    """{'signal' (, 'harmonic', 'noise')} numpy [B, T] from the kernels, through ops with explicit noise"""
    s = inp["synth"]
    f0 = inp["f0"].to(DEV)
    c = syn.split_views(inp["dense"].to(DEV), R.SPLITS[s])
    nz = inp["noise"].to(DEV)
    with torch.no_grad():
        if s == "superfast":
            ws, _ = ops.superfast_scan(f0, P, SR)
            out = (ops.superfast_synth(ws, c["harmonic_magnitude"], c["harmonic_phase"], c["noise_magnitude"],
                                       c["noise_phase"], P, WIN, noise_in=nz),)
        else:
            fph, _ = ops.phase_scan(f0, P, SR, infer=infer)
            if s == "sins":
                out = ops.sins_synth(f0, fph, c["amplitudes"], c["group_delay"], c["noise_magnitude"], P, SR,
                                     noise_in=nz, infer=infer)
            elif s == "combsub":
                out = ops.combsub_synth(f0, fph, c["group_delay"], c["harmonic_magnitude"], c["noise_magnitude"], P, SR,
                                        noise_in=nz, infer=infer)
            else:
                comb = ops.comb_source(f0, fph, P, SR, infer=infer)
                out = (ops.combsubfast_filter(comb, c["harmonic_magnitude"], c["harmonic_phase"], c["noise_magnitude"],
                                              P, noise_in=nz),)
    return {k: v.cpu().numpy() for k, v in zip(R.outputs_of(s), out)}


def check(tag, got, ref32, truth, rms_factor=RMS_FACTOR, max_factor=MAX_FACTOR):
    """record the three errors and assert the criterion of the module docstring for one output"""
    assert np.isfinite(got).all(), tag
    e = R.forward_errors(got, ref32, truth)
    report.record("regimes_forward/" + tag, **R.summary(e))
    bad = R.within_budget(e, rms_factor, max_factor)
    assert not bad, (tag, bad)


def compare_synth(tag, inp, infer):
    truth = R.truth_forward(inp)
    with torch.no_grad():
        ref = R.port_forward(inp, infer=infer)
    got = gpu_forward(inp, infer)
    for key in R.outputs_of(inp["synth"]):
        check("%s_%s" % (tag, key), got[key], ref[key].numpy(), truth[key])
    if inp["synth"] in R.HAS_PARTS:
        mix = got["harmonic"].astype(np.float64) + got["noise"]
        assert np.abs(got["signal"] - mix).max() <= 1e-6 * max(np.abs(mix).max(), 1e-30), tag


@pytest.mark.parametrize("case", R.TABLE, ids=R.CASE_IDS)
@pytest.mark.parametrize("synth,infer", MODES, ids=["%s-%s" % (s, "infer" if i else "train") for s, i in MODES])
def test_synthesizer_at_regime(synth, infer, case):
    inp = R.build(synth, *case)
    compare_synth("%s_%s_%s" % (synth, "infer" if infer else "train", "-".join(case)), inp, infer)


# ---------------------------------------------------------------------------------------------- SineGen
def _sinegen_inputs(pitch):
    B, nF, dim = (3, 48, 9) if pitch == "onsets" else (2, 24, 9)
    f0 = R.PITCH[pitch](B, nF, 31)[..., 0].contiguous()
    g = torch.Generator().manual_seed(32)
    ri = torch.rand(dim, generator=g)
    ri[0] = 0
    noise = torch.randn(B, nF * P, dim, generator=g)
    w, b = torch.randn(1, dim, generator=g) * 0.3, 0.05
    truth = cf.sinegen(f0.numpy(), P, SR, ri.numpy(), noise.numpy())
    merged = np.tanh(truth @ w.numpy().astype(np.float64).T + b)
    with torch.no_grad():
        ref = tp.source_module_forward(f0, P, SR, w, torch.tensor([b]), dim - 1, rand_ini=ri.reshape(1, 1, -1), noise=noise)
    return f0, ri, noise, w, b, truth, merged, ref


@pytest.mark.parametrize("impl", ["auto", "v1", "v2", "v2p"])
@pytest.mark.parametrize("pitch", list(R.PITCH))
def test_sinegen_and_source_module_at_pitch_regime(pitch, impl):
    f0, ri, noise, w, b, truth, merged, ref = _sinegen_inputs(pitch)
    try:
        ops.set_sinegen_impl(impl)
        got = ops.sinegen(f0.to(DEV), P, SR, 9, ri, noise_in=noise.to(DEV)).cpu().numpy()
        got_m = ops.source_module(f0.to(DEV), P, SR, 9, ri, w, b, noise_in=noise.to(DEV)).cpu().numpy()
    finally:
        ops.set_sinegen_impl("auto")
    check("sinegen_%s_%s" % (impl, pitch), got, ref["sines"].numpy(), truth)
    check("source_module_%s_%s" % (impl, pitch), got_m, ref["out"].numpy(), merged)


# ---------------------------------------------------------------------------------------------- stages
@pytest.mark.parametrize("case", STAGE_CASES, ids=["%s-%s" % c for c in STAGE_CASES])
@pytest.mark.parametrize("infer", [True, False], ids=["infer", "train"])
def test_stage_kernels_at_regime(case, infer):
    """phase_scan, sins_bank, comb_source, ir_build in its three modes and ltv_fir on their own against the stages of
    the same truth, so that a failure of a synthesizer names its kernel.  Each FIR is fed the float64 stage before it
    rounded to fp32, and compared with the float64 FIR of exactly that input."""
    tag = "stage_%s_%s_" % ("infer" if infer else "train", "-".join(case))
    sins, comb = R.build("sins", *case), R.build("combsub", *case)
    comb["f0"] = sins["f0"]
    f0 = sins["f0"].to(DEV)
    t_s, t_c = R.truth_forward(sins), R.truth_forward(comb)
    with torch.no_grad():
        r_s, r_c = R.port_forward(sins, infer=infer), R.port_forward(comb, infer=infer)
    cs, cc = (syn.split_views(i["dense"].to(DEV), R.SPLITS[i["synth"]]) for i in (sins, comb))

    fph, phase_frames = ops.phase_scan(f0, P, SR, infer=infer)
    wrap = lambda d: (d + np.pi) % (2 * np.pi) - np.pi
    want = 2 * np.pi * t_s["x"][:, ::P]
    d_gpu = wrap(phase_frames[..., 0].cpu().numpy().astype(np.float64) - want)
    d_ref = wrap(r_s["phase_frames"][..., 0].numpy().astype(np.float64) - want)
    report.record("regimes_forward/" + tag + "phase_frames", gpu_vs_truth=np.abs(d_gpu).max(),
                  ref32_vs_truth=np.abs(d_ref).max())
    assert np.abs(d_gpu).max() <= max(2e-6, RMS_FACTOR * np.abs(d_ref).max())

    check(tag + "sins_bank", ops.sins_bank(f0, fph, cs["amplitudes"], P, SR, infer=infer).cpu().numpy(),
          r_s["sinusoids"].numpy(), t_s["sinusoids"])
    check(tag + "comb_source", ops.comb_source(f0, fph, P, SR, infer=infer).cpu().numpy(), r_c["comb"].numpy(), t_c["comb"])
    irs = {}
    for name, ctrl, mode, ref, truth in (
            ("ir_allpass", cs["group_delay"], ops.IR_ALLPASS, r_s["ir_allpass"], t_s["ir_allpass"]),
            ("ir_noise", cs["noise_magnitude"], ops.IR_MAG_HANN, r_s["ir_noise"], t_s["ir_noise"]),
            ("ir_harmonic", cc["harmonic_magnitude"], ops.IR_MAG_DYNAMIC, r_c["ir_harmonic"], t_c["ir_harmonic"])):
        B, nF, L = truth.shape
        for impl in ("cuda", "tc"):
            try:
                ops.set_ir_impl(impl)
                irs[name] = ops.ir_build(ctrl, mode, SR, f0_frames=f0 if mode == ops.IR_MAG_DYNAMIC else None)
            finally:
                ops.set_ir_impl("auto")
            check(tag + name + "_" + impl, irs[name].cpu().numpy().reshape(B, nF * L), ref.numpy().reshape(B, nF * L),
                  truth.reshape(B, nF * L))
    for name, x, ir in (("fir_allpass", t_s["sinusoids"], t_s["ir_allpass"]),
                        ("fir_harmonic", t_c["allpassed"], t_c["ir_harmonic"])):
        x32, ir32 = torch.from_numpy(x).float(), torch.from_numpy(ir).float().contiguous()
        truth = cf.ltv_fir(x32.numpy(), ir32.numpy(), P)
        ref = tp.ltv_fir(x32, ir32).numpy()
        for impl in ("cuda", "tc", "fft"):
            try:
                ops.set_fir_impl(impl)
                got = ops.ltv_fir(x32.to(DEV), ir32.to(DEV), P).cpu().numpy()
            finally:
                ops.set_fir_impl("auto")
            check(tag + name + "_" + impl, got, ref, truth)


# ---------------------------------------------------------------------------------------------- variants
@pytest.mark.parametrize("case", STAGE_CASES, ids=["%s-%s" % c for c in STAGE_CASES])
@pytest.mark.parametrize("setter,impl", [("set_sins_impl", "split"), ("set_sins_impl", "fused"),
                                         ("set_sins_impl", "spectrum"), ("set_fir_impl", "cuda"), ("set_fir_impl", "tc"),
                                         ("set_fir_impl", "fft"), ("set_ir_impl", "cuda"), ("set_ir_impl", "tc")])
def test_selectable_variants_at_regime(setter, impl, case):
    """every variant a user can select computes the same thing at these inputs, to the same criterion"""
    synths = ("sins",) if setter == "set_sins_impl" else ("sins", "combsub")
    for synth in synths:
        inp = R.build(synth, *case)
        for infer in (True, False):
            try:
                getattr(ops, setter)(impl)
                compare_synth("variant_%s_%s_%s_%s_%s" % (setter[4:], impl, synth, "infer" if infer else "train",
                                                          "-".join(case)), inp, infer)
            finally:
                getattr(ops, setter)("auto")


# ---------------------------------------------------------------------------------------------- long rows
def _long_row(synth):
    nF = 5168                                                        # 60 s
    f0 = R.onsets(1, nF, seed=71)
    dense, views = R.trained(1, nF, R.SPLITS[synth], seed=72)
    g = torch.Generator().manual_seed(73)
    noise = torch.randn(1, nF * P, generator=g) if synth == "superfast" else torch.rand(1, nF * P, generator=g) * 2 - 1
    return {"synth": synth, "B": 1, "nF": nF, "f0": f0, "dense": dense, "ctrls": views, "noise": noise}


@pytest.mark.parametrize("synth", list(R.SPLITS))
def test_one_minute_row(synth):
    """B = 1, 60 s (nothing else runs longer than 10 s; an inference segment is as long as the singer goes without a
    pause), voiced / unvoiced runs, trained controls: the whole row against the fp32 port, and its last 2 s against the
    float64 closed form of the last 2 s.  The truth of a tail needs the phase at its start: float64 frame sums."""
    inp = _long_row(synth)
    with torch.no_grad():
        ref = R.port_forward(inp, infer=True)["signal"].numpy()
    got = gpu_forward(inp, True)["signal"]
    assert np.isfinite(got).all()
    e = R.rms_rows(got - ref)[0]
    scale = max(1.0, R.rms_rows(ref)[0] / 0.01)
    report.record("regimes_forward/long_%s" % synth, gpu_vs_ref32=e, gpu_vs_ref32_max=np.abs(got - ref).max(),
                  ref32_rms=R.rms_rows(ref)[0])
    assert e <= 2e-6 * scale, (synth, e)
    # the last 2 s against float64: everything but the source is local in time (FIR / STFT reach < 4 frames), and the
    # closed-form sources take the whole f0 row cheaply
    tail = 172
    f0 = inp["f0"].numpy()
    if synth == "superfast":
        rad, s_up = cf.superfast_phase(f0, SR, P)
        src = np.sinc(rad / (s_up + 1e-5)).reshape(1, -1)
    else:
        x = cf.phase_cycles(f0, SR, P).astype(np.float32).astype(np.float64)
        src = x if synth == "sins" else np.sinc(SR * x / (cf.upsample(f0, P)[..., 0] + 1e-3))
    lo = inp["nF"] - tail - 8                                         # 8 frames of run-in, dropped below
    c = {k: v.numpy()[:, lo:] for k, v in inp["ctrls"].items()}
    nz, f0t, srct = inp["noise"].numpy()[:, lo * P:], f0[:, lo:], src[:, lo * P:]
    if synth == "sins":
        sinus = cf.sinusoid_bank(srct, cf.harmonic_amplitudes(c["amplitudes"], f0t, SR), P)
        truth = cf.ltv_fir(sinus, cf.impulse_response(cf.allpass_spectrum(c["group_delay"]), "none"), P) + \
            cf.ltv_fir(nz, cf.impulse_response(np.exp(c["noise_magnitude"].astype(np.float64)) / 128.0, "hann"), P)
    elif synth == "combsub":
        ap = cf.ltv_fir(srct, cf.impulse_response(cf.allpass_spectrum(c["group_delay"]), "none"), P)
        hw = 1.5 * SR / (f0t.astype(np.float64) + 1e-3)
        truth = cf.ltv_fir(ap, cf.impulse_response(np.exp(c["harmonic_magnitude"].astype(np.float64)), "dynamic", hw), P) + \
            cf.ltv_fir(nz, cf.impulse_response(np.exp(c["noise_magnitude"].astype(np.float64)) / 128.0, "hann"), P)
    else:
        truth = _filter_truth(synth, srct, c, nz)
    keep = slice(8 * P, None)
    check("long_tail_%s" % synth, got[:, lo * P:][:, keep], ref[:, lo * P:][:, keep], truth[:, keep])


def _filter_truth(synth, comb, c, noise):
    """the STFT-domain filters of CombSubFast / CombSubSuperFast in float64 on a given comb (oracle.closed_form's
    arithmetic with the source passed in)"""
    hold = lambda z: np.concatenate([z, z[:, -1:, :]], axis=1)
    c = {k: np.asarray(v, np.float64) for k, v in c.items()}
    if synth == "superfast":
        h_src = hold(np.exp(c["harmonic_magnitude"] + 1j * np.pi * c["harmonic_phase"]))
        h_noise = hold(np.exp(c["noise_magnitude"] + 1j * np.pi * c["noise_phase"]) / 128.0)
        spec = cf.stft_frames(comb, WIN, P) * h_src + cf.stft_frames(np.asarray(noise, np.float64), WIN, P) * h_noise
        return cf.istft_frames(spec, WIN, P)
    B, T = comb.shape
    nF, N = T // P, 2 * P
    w = np.sqrt(0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N))
    h_src = hold(np.exp(c["harmonic_magnitude"] + 1j * np.pi * c["harmonic_phase"]))
    h_noise = hold(np.exp(c["noise_magnitude"]) / 128.0)
    pad = lambda z: np.concatenate([np.zeros((B, P)), np.asarray(z, np.float64), np.zeros((B, P))], axis=1)
    cp, zp = pad(comb), pad(noise)
    out = np.zeros((B, T + 2 * P))
    for q in range(nF + 1):
        seg = slice(q * P, q * P + N)
        spec = np.fft.rfft(cp[:, seg] * w, N) * h_src[:, q] + np.fft.rfft(zp[:, seg] * w, N) * h_noise[:, q]
        out[:, seg] += np.fft.irfft(spec, N) * w
    return out[:, P:-P]


def test_one_minute_sinegen_row():
    nF, dim = 5168, 9
    f0 = R.onsets(1, nF, seed=81)[..., 0].contiguous()
    g = torch.Generator().manual_seed(82)
    ri = torch.rand(dim, generator=g)
    ri[0] = 0
    noise = torch.randn(1, nF * P, dim, generator=g)
    with torch.no_grad():
        ref = tp.sinegen_forward(f0, P, SR, dim - 1, rand_ini=ri.reshape(1, 1, -1), noise=noise)["out"].numpy()
    truth = cf.sinegen(f0.numpy(), P, SR, ri.numpy(), noise.numpy())
    got = ops.sinegen(f0.to(DEV), P, SR, dim, ri, noise_in=noise.to(DEV)).cpu().numpy()
    check("long_sinegen", got, ref, truth)
