"""The wgmma (tensor-core, 3xTF32) time-varying FIR against the CUDA-core kernel, the
one-thread-per-sample kernel and the oracle.  It is not the default dispatch (it is correct but
operand-bandwidth bound, see ltv_fir_tc.cu); these tests keep it honest, including one full Sins
forward through it."""
import pytest
import torch

from ddsp_svc_b200 import ops, synthetic as syn
from tests import report, util
from tests.golden import cases as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P = G.SR, G.P


@pytest.fixture(autouse=True)
def _restore_impl():
    yield
    ops.set_fir_impl("auto")


@pytest.mark.parametrize("name", ["sins_b2_f24_h128", "sins_b1_f2_h128", "sins_b3_f1_h128", "sins_b1_f7_h33"])
def test_tc_vs_cuda_vs_oracle_510_taps(name):
    inp = G.build_inputs(name)
    ref = util.port_outputs(name, inp)
    x = ref["sinusoids"].to(DEV)
    ir = ref["ir_allpass"].to(DEV).contiguous()
    ops.set_fir_impl("tc")
    y_tc = ops.ltv_fir(x, ir, P).cpu()
    ops.set_fir_impl("cuda")
    y_cc = ops.ltv_fir(x, ir, P).cpu()
    e_tc, e_cc = util.rms(y_tc - ref["harmonic"]), util.rms(y_cc - ref["harmonic"])
    report.record("fir_tc/" + name, tc_rms=e_tc, cuda_rms=e_cc, tc_vs_cuda_max=(y_tc - y_cc).abs().max().item(),
                  ref_rms=util.rms(ref["harmonic"]))
    assert e_tc < 5e-7 and e_cc < 5e-7


def test_tc_1022_taps_two_segments():
    name = "combsub_b2_f24"
    inp = G.build_inputs(name)
    ref = util.port_outputs(name, inp)
    x, ir = ref["allpassed"].to(DEV), ref["ir_harmonic"].to(DEV).contiguous()
    ops.set_fir_impl("tc")
    y = ops.ltv_fir(x, ir, P).cpu()
    e = util.rms(y - ref["harmonic"])
    report.record("fir_tc/1022", rms=e, ref_rms=util.rms(ref["harmonic"]))
    assert e < 1e-6


def test_tc_full_size_vs_generic_and_noise_modes():
    B, nF = 32, 861
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(B, nF * P, generator=g) * 2 - 1).to(DEV)
    ir = (torch.randn(B, nF, 510, generator=g) * 0.05).to(DEV)
    ops.set_fir_impl("tc")
    y_tc = ops.ltv_fir(x, ir, P)
    y_g = ops.ltv_fir(x, ir, P, generic=True)
    scale = y_g.pow(2).mean().sqrt().item()
    e = (y_tc - y_g).pow(2).mean().sqrt().item()
    report.record("fir_tc/full", rel_rms=e / scale, max=(y_tc - y_g).abs().max().item(), scale=scale)
    assert e / scale < 2e-5     # the fp32 tensor-core accumulator truncates: ~5e-6 after 390 accumulation steps
    # in-kernel noise: identical stream in both implementations (same Philox keying)
    ident = torch.zeros(2, 16, 510, device=DEV); ident[:, :, 255] = 1.0
    a = ops.ltv_fir(None, ident, P, seed=7)
    ops.set_fir_impl("cuda")
    b = ops.ltv_fir(None, ident, P, seed=7)
    assert (a - b).abs().max().item() < 1e-6


def test_sins_forward_through_the_tensor_core_fir():
    from ddsp_svc_b200 import FixedControls, Sins
    name = "sins_b2_f24_h128"
    inp = G.build_inputs(name)
    gold = util.load_golden(name)
    case = inp["case"]
    ctrls = syn.split_views(inp["dense"].to(DEV), G.split_map(case))
    model = Sins(SR, P, case["H"], case["Ma"], case["Mn"], unit2ctrl=FixedControls(ctrls, None)).to(DEV)
    ops.set_fir_impl("tc")
    with torch.no_grad():
        signal, _, (harm, nz) = model(None, inp["f0"].to(DEV), None, noise=inp["noise"].to(DEV))
    e = util.rms(signal.cpu().numpy() - gold["signal"])
    report.record("fir_tc/sins_forward", signal_err=e)
    assert e < 2e-6
    assert torch.equal(signal, harm + nz)      # red.add of exactly two addends is order independent
