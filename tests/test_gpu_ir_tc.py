"""The impulse-response builders against the float64 reference of test_gpu_kernel_variants.ir_reference, per tap
within HEADROOM * EPS * sum_m |w_m H_m| plus the worst-case budget of the accumulation over the bins: the wgmma
(3xTF32) kernel with 32-row and 64-row CTAs, the CUDA-core kernel (forced, and as the automatic fallback above the
tensor-core limits, with more than 48 KB of shared memory), for all three modes, n_mag from 2 to 1025, strided
controls, saturating controls and f0 from 0 to near Nyquist.  Also the constant table buffer both kernels read, value
by value."""
import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib, ops
from tests import report
from tests.test_gpu_kernel_variants import (_check, assert_launched, cc_table_floats, cc_table_layout, dft_value,
                                            ir_reference, profiled, tc_image_from_values)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 44100


@pytest.fixture(autouse=True)
def _restore():
    yield
    ops.set_ir_impl("auto")


def _controls(mode, B, nF, M, seed):
    """Seeded raw controls as a device view with an odd frame stride.  Even frames: the model's usual range.  Odd
    frames: all-pass controls saturated (|c| in [10, 30], mostly positive, so the phase runs up to ~0.8 pi per bin and
    tanh is exactly +-1 in fp32), magnitude controls uniform in [-30, 12].  Also f0 [B, nF, 1]: 60-760 Hz, one 0 Hz
    frame, and every third frame of the second utterance near Nyquist (half widths of ~3 taps)."""
    g = torch.Generator().manual_seed(seed * 100003 + M * 7 + mode * 1009)
    width = M + 13 if (M + 13) % 2 else M + 14
    mu, sd = {ops.IR_ALLPASS: (0.0, 0.3), ops.IR_MAG_HANN: (-3.0, 0.5), ops.IR_MAG_DYNAMIC: (-2.0, 0.5)}[mode]
    dense = torch.randn(B, nF, width, generator=g) * sd + mu
    odd = dense[:, 1::2]
    if mode == ops.IR_ALLPASS:
        sign = torch.where(torch.rand(odd.shape, generator=g) < 0.85, 1.0, -1.0)
        odd.copy_(sign * (10.0 + 20.0 * torch.rand(odd.shape, generator=g)))
    else:
        odd.copy_(-30.0 + 42.0 * torch.rand(odd.shape, generator=g))
    f0 = torch.rand(B, nF, 1, generator=g) * 700 + 60
    f0[0, min(3, nF - 1)] = 0.0
    if B > 1:
        f0[1, ::3] = 20000.0 + 2000.0 * torch.rand(f0[1, ::3].shape, generator=g)
    c = dense.to(DEV)[..., 5:5 + M]
    assert c.stride(1) % 2 == 1
    return c, f0


def _build(c, mode, f0):
    return ops.ir_build(c, mode, SR, f0_frames=f0.to(DEV) if mode == ops.IR_MAG_DYNAMIC else None).cpu().numpy()


@pytest.mark.parametrize("mode,n_mag", [(ops.IR_ALLPASS, 256), (ops.IR_MAG_HANN, 256), (ops.IR_MAG_DYNAMIC, 512),
                                         (ops.IR_ALLPASS, 65), (ops.IR_MAG_HANN, 129), (ops.IR_MAG_DYNAMIC, 256),
                                         (ops.IR_ALLPASS, 9), (ops.IR_MAG_HANN, 2),
                                         (ops.IR_ALLPASS, 2), (ops.IR_ALLPASS, 3), (ops.IR_MAG_DYNAMIC, 3),
                                         (ops.IR_ALLPASS, 33), (ops.IR_MAG_HANN, 33), (ops.IR_MAG_DYNAMIC, 33),
                                         (ops.IR_MAG_HANN, 101), (ops.IR_MAG_HANN, 512)])
def test_ir_tc_matches_oracle_and_cuda(mode, n_mag):
    """n_mag 2, 3, odd sizes, 33 (17 columns: one past a 16-column tile) and the largest the tensor cores take
    (256 all-pass, 512 magnitude)."""
    B, nF = 3, 50                       # 150 frames: five CTAs of 32 rows (a single wave), the last one partial
    c, f0 = _controls(mode, B, nF, n_mag, seed=0)
    ref, bound = ir_reference(c.cpu().numpy(), mode, f0.numpy())
    bound_tc = ir_reference(c.cpu().numpy(), mode, f0.numpy(), tensor_cores=True)[1]
    ops.set_ir_impl("cuda")
    ir_cc, cc_names = profiled(_build, c, mode, f0)
    ops.set_ir_impl("tc")
    ir_tc, tc_names = profiled(_build, c, mode, f0)
    _check("ir_tc/mode%d_m%d/cuda" % (mode, n_mag), ir_cc, ref, bound)
    _check("ir_tc/mode%d_m%d/tc" % (mode, n_mag), ir_tc, ref, bound_tc)
    assert_launched(cc_names, "ir_build_kernel<%d>" % mode)
    assert_launched(tc_names, "ir_build_tc_kernel<%d, 32>" % mode)


@pytest.mark.parametrize("mode,n_mag", [(ops.IR_ALLPASS, 256), (ops.IR_MAG_HANN, 256), (ops.IR_MAG_DYNAMIC, 512)])
def test_ir_tc_64_row_ctas(mode, n_mag):
    """More than one wave of 32-row CTAs switches to 64 rows per CTA: 32 * SMs + 40 frames (rounded up to B = 3
    utterances of equal length, so utterance boundaries fall inside CTAs), not a multiple of 64, so the last CTA is
    partial."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    B = 3
    nF = (32 * sms + 40 + B - 1) // B
    assert B * nF > 32 * sms and (B * nF) % 64 != 0
    c, f0 = _controls(mode, B, nF, n_mag, seed=1)
    ref, bound = ir_reference(c.cpu().numpy(), mode, f0.numpy(), tensor_cores=True)
    ir, names = profiled(_build, c, mode, f0)
    _check("ir_tc64/mode%d_m%d" % (mode, n_mag), ir, ref, bound, frames=B * nF)
    assert_launched(names, "ir_build_tc_kernel<%d, 64>" % mode)


@pytest.mark.parametrize("mode,n_mag", [(ops.IR_ALLPASS, 257), (ops.IR_ALLPASS, 385), (ops.IR_ALLPASS, 1025),
                                         (ops.IR_MAG_HANN, 513), (ops.IR_MAG_HANN, 1025),
                                         (ops.IR_MAG_DYNAMIC, 513), (ops.IR_MAG_DYNAMIC, 769),
                                         (ops.IR_MAG_DYNAMIC, 1025)])
def test_ir_auto_falls_back_to_cuda_cores(mode, n_mag):
    """Above the tensor-core limit (all-pass 256, magnitude 512 bins) 'auto' builds on CUDA cores and 'tc' refuses.
    From 385 (all-pass) / 769 (magnitude) bins that kernel needs more than 48 KB of dynamic shared memory."""
    B, nF = 2, 21                       # 42 frames: three CTAs of 16, the last one partial
    c, f0 = _controls(mode, B, nF, n_mag, seed=2)
    ref, bound = ir_reference(c.cpu().numpy(), mode, f0.numpy())
    ir, names = profiled(_build, c, mode, f0)
    _check("ir_auto/mode%d_m%d" % (mode, n_mag), ir, ref, bound)
    ops.set_ir_impl("tc")
    with pytest.raises(ValueError, match="tensor-core path does not support"):
        _build(c, mode, f0)
    assert_launched(names, "ir_build_kernel<%d>" % mode)


@pytest.mark.parametrize("n_mag", [2, 3, 33, 256, 257, 512, 1025])
def test_dft_table_buffer(n_mag):
    """ops.dft_tables: every CUDA-core table value within one fp32 ulp of cos / sin(2 pi m t / L), and the tensor-core
    operand image (layout documented in ir_build_tc.cu) holding the exact tf32 hi / lo split of those stored values,
    zeros in its padding."""
    tab = ops.dft_tables(n_mag, DEV).cpu().numpy()
    assert tab.size * 4 == _lib.lib().b2d_dft_tables_bytes(n_mag)
    m, t, is_sin = cc_table_layout(n_mag)
    cc = tab[:m.size]
    exact = dft_value(m, t, is_sin, n_mag)
    err = np.abs(cc.astype(np.float64) - exact)
    ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
    img = tab[cc_table_floats(n_mag):]
    want = tc_image_from_values(n_mag, cc)
    report.record("dft_tables/m%d" % n_mag, max_err_over_ulp=float((err / (ulp + 1e-15)).max()),
                  image_mismatches=int((img.view(np.uint32) != want.view(np.uint32)).sum()))
    assert np.all(err <= ulp + 1e-15)
    assert img.size == want.size
    assert np.array_equal(img.view(np.uint32), want.view(np.uint32))
