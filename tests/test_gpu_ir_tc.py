"""The wgmma (3xTF32) impulse-response builder against the CUDA-core kernel and the oracle, for
all three modes and several n_mag (including sizes that need column / K padding)."""
import math

import pytest
import torch

from ddsp_svc_b200 import ops
from oracle import torch_port as tp
from tests import report, util

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 44100


@pytest.fixture(autouse=True)
def _restore():
    yield
    ops.set_ir_impl("auto")


def _oracle_ir(c, mode, f0):
    with torch.no_grad():
        if mode == ops.IR_ALLPASS:
            gd = math.pi * torch.tanh(c)
            return tp.impulse_response(torch.exp(1.j * torch.cumsum(gd, dim=-1)), "none")
        if mode == ops.IR_MAG_HANN:
            mag = torch.exp(c) / 128
            return tp.impulse_response(torch.complex(mag, torch.zeros_like(mag)), "hann")
        mag = torch.exp(c)
        return tp.impulse_response(torch.complex(mag, torch.zeros_like(mag)), "dynamic",
                                   1.5 * torch.tensor(SR) / (f0 + 1e-3))


@pytest.mark.parametrize("mode,n_mag", [(ops.IR_ALLPASS, 256), (ops.IR_MAG_HANN, 256), (ops.IR_MAG_DYNAMIC, 512),
                                         (ops.IR_ALLPASS, 65), (ops.IR_MAG_HANN, 129), (ops.IR_MAG_DYNAMIC, 256),
                                         (ops.IR_ALLPASS, 9), (ops.IR_MAG_HANN, 2)])
def test_ir_tc_matches_oracle_and_cuda(mode, n_mag):
    B, nF = 3, 50                       # 150 frames: two CTAs of 128 rows, the second partly empty
    g = torch.Generator().manual_seed(n_mag * 7 + mode)
    mu, sd = {ops.IR_ALLPASS: (0.0, 0.3), ops.IR_MAG_HANN: (-3.0, 0.5), ops.IR_MAG_DYNAMIC: (-2.0, 0.5)}[mode]
    c = torch.randn(B, nF, n_mag, generator=g) * sd + mu
    f0 = torch.rand(B, nF, 1, generator=g) * 700 + 60
    f0[0, 3] = 0.0
    ref = _oracle_ir(c, mode, f0)
    f0d = f0.to(DEV) if mode == ops.IR_MAG_DYNAMIC else None
    ops.set_ir_impl("cuda")
    ir_cc = ops.ir_build(c.to(DEV), mode, SR, f0_frames=f0d).cpu()
    ops.set_ir_impl("tc")
    ir_tc = ops.ir_build(c.to(DEV), mode, SR, f0_frames=f0d).cpu()
    peak = ref.abs().max().item()
    e_tc, e_cc = (ir_tc - ref).abs().max().item(), (ir_cc - ref).abs().max().item()
    report.record("ir_tc/mode%d_m%d" % (mode, n_mag), tc_max=e_tc, cuda_max=e_cc, peak=peak,
                  tc_rms=util.rms(ir_tc - ref), cuda_rms=util.rms(ir_cc - ref))
    tol = 5e-5 if mode == ops.IR_ALLPASS else 2e-6 * max(peak, 1e-3)
    assert e_cc < tol, ("cuda", e_cc, tol)
    assert e_tc < tol, ("tc", e_tc, tol)
    assert util.rms(ir_tc - ref) < 5e-6 * max(1.0, peak)
