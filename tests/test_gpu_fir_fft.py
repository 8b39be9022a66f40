"""The FFT-domain time-varying FIR (csrc/ltv_fir_fft.cu, ops.set_fir_impl("fft")) against the CUDA-core kernel, the
oracle and the goldens, including full Sins / CombSub forwards through it.

It is the automatic dispatch for block size 512 and <= 1024 taps (faster than the direct form), so every Sins /
CombSub test also runs through it; these tests compare it explicitly with the direct form."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import CombSub, FixedControls, Sins, ops, synthetic as syn
from tests import report, util
from tests.golden import cases as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P = G.SR, G.P


@pytest.fixture(autouse=True)
def _restore_impl():
    yield
    ops.set_fir_impl("auto")


@pytest.mark.parametrize("name", ["sins_b2_f24_h128", "sins_b1_f2_h128", "sins_b3_f1_h128", "sins_b1_f7_h33",
                                  "sins_b1_f12_h40_m65_initphase"])
def test_fft_vs_cuda_vs_oracle(name):
    inp = G.build_inputs(name)
    ref = util.port_outputs(name, inp)
    x, ir = ref["sinusoids"].to(DEV), ref["ir_allpass"].to(DEV).contiguous()
    ops.set_fir_impl("fft")
    y_f = ops.ltv_fir(x, ir, P).cpu()
    ops.set_fir_impl("cuda")
    y_c = ops.ltv_fir(x, ir, P).cpu()
    e_f, e_c = util.rms(y_f - ref["harmonic"]), util.rms(y_c - ref["harmonic"])
    report.record("fir_fft/" + name, fft_rms=e_f, cuda_rms=e_c, max_diff=(y_f - y_c).abs().max().item(),
                  ref_rms=util.rms(ref["harmonic"]))
    assert e_f < 2e-7 and (y_f - y_c).abs().max().item() < 5e-6


@pytest.mark.parametrize("name", [n for n, c in G.CASES.items() if c["kind"] in ("sins", "combsub")])
def test_forward_through_fft_fir_matches_golden(name):
    inp = G.build_inputs(name)
    gold = util.load_golden(name)
    case = inp["case"]
    ctrl = syn.split_views(inp["dense"].to(DEV), G.split_map(case))
    fixed = FixedControls(ctrl, torch.zeros(1, device=DEV))
    if case["kind"] == "sins":
        model = Sins(SR, P, case["H"], case["Ma"], case["Mn"], unit2ctrl=fixed).to(DEV)
    else:
        model = CombSub(SR, P, case["Ma"], case["Mh"], case["Mn"], unit2ctrl=fixed).to(DEV)
    kw = {"initial_phase": inp["initial_phase"].to(DEV)} if "initial_phase" in inp else {}
    ops.set_fir_impl("fft")
    with torch.no_grad():
        signal, _, (harm, noise) = model(None, inp["f0"].to(DEV), None, noise=inp["noise"].to(DEV), **kw)
    e = util.rms(signal.cpu().numpy() - gold["signal"])
    rec = {"signal_rms": e}
    for key, t in (("harmonic", harm), ("noise", noise)):
        if key in gold:
            rec[key + "_rms"] = util.rms(t.cpu().numpy() - gold[key])
            assert rec[key + "_rms"] < 2e-6
    report.record("fir_fft_forward/" + name, **rec)
    assert e < 2e-6


def test_fft_1022_taps_uses_the_2048_point_transform():
    name = "combsub_b2_f24"
    ref = util.port_outputs(name, G.build_inputs(name))
    x, ir = ref["allpassed"].to(DEV), ref["ir_harmonic"].to(DEV).contiguous()
    ops.set_fir_impl("fft")
    y = ops.ltv_fir(x, ir, P).cpu()
    e = util.rms(y - ref["harmonic"])
    report.record("fir_fft/1022", rms=e, ref_rms=util.rms(ref["harmonic"]))
    assert e < 2e-6 * util.rms(ref["harmonic"]) + 1e-9


def test_fft_full_size_vs_cuda_and_in_kernel_noise():
    B, nF = 32, 861
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(B, nF * P, generator=g) * 2 - 1).to(DEV)
    ir = (torch.randn(B, nF, 510, generator=g) * 0.05).to(DEV)
    ops.set_fir_impl("fft")
    y_f = ops.ltv_fir(x, ir, P)
    n_f = ops.ltv_fir(None, ir, P, seed=11, utterance_offset=3)
    ops.set_fir_impl("cuda")
    y_c = ops.ltv_fir(x, ir, P)
    n_c = ops.ltv_fir(None, ir, P, seed=11, utterance_offset=3)
    scale = y_c.pow(2).mean().sqrt().item()
    e = (y_f - y_c).pow(2).mean().sqrt().item()
    en = (n_f - n_c).pow(2).mean().sqrt().item()
    report.record("fir_fft_full", rel_rms=e / scale, noise_rel_rms=en / scale)
    # two fp32 evaluations of the same sum with white (unwindowed) impulse responses: equal to fp32 round-off;
    # same Philox stream in both kernels
    assert e < 3e-6 * scale and en < 3e-6 * scale
