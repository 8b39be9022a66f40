"""The "packed" and "scalar" instantiations of the FFT kernels (ops.set_fft_arith) against each other.

Hopper has no packed FP32 add, so both instantiations perform the same scalar complex additions and their outputs are
identical: the test checks that."""
import pytest
import torch

from ddsp_svc_b200 import CombSubFast, CombSubSuperFast, FixedControls, Sins, ops, synthetic as syn
from tests import report
from tests.golden import cases as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P = G.SR, G.P


@pytest.fixture(autouse=True)
def _restore():
    yield
    ops.set_fft_arith("packed")          # the library default


def _model(kind, B, nF):
    if kind == "sins":
        sm = syn.sins_split_map(128, 256, 256)
        make = lambda fixed: Sins(SR, P, 128, 256, 256, unit2ctrl=fixed)
    elif kind == "superfast":
        sm = syn.superfast_split_map(2048)
        make = lambda fixed: CombSubSuperFast(SR, P, 2048, unit2ctrl=fixed)
    else:
        sm = syn.combsubfast_split_map(P)
        make = lambda fixed: CombSubFast(SR, P, unit2ctrl=fixed)
    dense = syn.make_ctrl(B, nF, sm, seed=3)[0].to(DEV)
    fixed = FixedControls(syn.split_views(dense, sm), None)
    return make(fixed).to(DEV)


@pytest.mark.parametrize("kind", ["sins", "superfast", "combsubfast"])
def test_packed_matches_scalar(kind):
    B, nF = 3, 70
    model = _model(kind, B, nF)
    f0 = syn.make_f0(B, nF, SR, P, seed=4, unvoiced_fraction=0.2).to(DEV)
    noise = (syn.normal_noise((B, nF * P), 5) if kind == "superfast" else syn.uniform_noise(B, nF * P, 5)).to(DEV)
    with torch.no_grad():
        ops.set_fft_arith("scalar")
        ref = model(None, f0, None, noise=noise)[0]
        ops.set_fft_arith("packed")
        got = model(None, f0, None, noise=noise)[0]
    scale = ref.pow(2).mean().sqrt().item()
    err = (got - ref).abs().max().item()
    report.record("fft_packed/" + kind, max_diff=err, ref_rms=scale, identical=bool(torch.equal(got, ref)))
    assert torch.equal(got, ref), err
