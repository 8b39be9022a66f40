"""CPU checks of the float64 references and table layouts that the GPU variant tests (test_gpu_kernel_variants.py,
test_gpu_ir_tc.py) compare the kernels with."""
import numpy as np
import pytest

from ddsp_svc_b200 import _lib, ops
from oracle import closed_form as cf
from tests.test_gpu_kernel_variants import (allpass_phase_bound, allpass_spectrum_fp32, cc_table_floats,
                                            cc_table_layout, dft_dims, dynamic_window_u, ir_reference, ir_weights,
                                            split_tf32, tc_accumulation_eps, tc_image_layout)


@pytest.mark.parametrize("M", [9, 257, 1025])
def test_allpass_fp32_phase_reference_within_its_bound(M):
    """The all-pass impulse response on the fp32 phase differs from the pure float64 one by at most
    sum_m w_m |dphi_m|, with dphi bounded per bin by allpass_phase_bound; saturated one-signed controls drive the
    phase to ~pi per bin (thousands of radians at 1025 bins), where the fp32 phase is off by up to half an ulp."""
    rng = np.random.default_rng(M)
    c = np.concatenate([rng.normal(0.0, 0.3, (3, M)), rng.uniform(10, 30, (2, M)),
                        rng.choice([-1.0, 1.0], (2, M), p=[0.15, 0.85]) * rng.uniform(10, 30, (2, M))])
    c = c.astype(np.float32)
    h32 = cf.impulse_response(allpass_spectrum_fp32(c), "none")
    h64 = cf.impulse_response(cf.allpass_spectrum(c), "none")
    bound = (ir_weights(M) * allpass_phase_bound(c)).sum(-1, keepdims=True) + 1e-12
    assert np.all(np.abs(h32 - h64) <= bound)
    if M == 1025:
        phi = np.cumsum(np.pi * np.tanh(c.astype(np.float64)), -1)
        assert np.abs(phi).max() > 3000      # the regime the fp32-phase reference exists for


def test_dynamic_window_decides_u_above_1_in_fp32():
    """At f0 = 696.3148 Hz and 512 bins, tap 606 has u = 95 / hw: exactly 1 in fp32 (window 0, as the reference's fp32
    torch computes it) but above 1 in float64 (window 1).  Elsewhere the window is closed_form's."""
    M, f0 = 512, np.float32(696.3148)
    u = dynamic_window_u(f0, M)
    hw = 1.5 * 44100 / (np.float64(f0) + 1e-3)
    assert 95 / hw > 1 and u[606] == 95 / hw
    rng = np.random.default_rng(1)
    spec = np.exp(rng.normal(-2, 0.5, (4, M)))
    f0s = np.array([[0.0], [150.0], [696.3148], [21000.0]], np.float32)
    h, _ = ir_reference(np.log(spec).astype(np.float32), ops.IR_MAG_DYNAMIC, f0s)
    want = cf.impulse_response(np.exp(np.log(spec).astype(np.float32).astype(np.float64)), "dynamic",
                               1.5 * 44100 / (f0s.astype(np.float64) + 1e-3))
    differ = np.argwhere(np.abs(h - want) > 1e-12 * np.abs(want).max())
    assert differ.tolist() == [[2, 606]]


def _decode(i, M):
    """scalar decode of image index i, spelled out from the layout comment of dft_image_kernel (ir_build_tc.cu)"""
    _, Nt, Ke, Ko = dft_dims(M)
    Npad = ((Nt + 15) // 16) * 16
    bblock = Npad * 8
    ch, rem = divmod(i, 8 * bblock)
    blk, inner = divmod(rem, bblock)
    half, r = divmod(inner, Npad * 4)
    n, e = divmod(r, 4)
    k = 8 * ch + 4 * half + e
    tab, lo = blk >> 1, blk & 1
    odd = tab >= 2
    valid = n < Nt and k < (Ko if odd else Ke)
    return 2 * k + odd, n, bool(tab & 1), bool(lo), valid


@pytest.mark.parametrize("M", [2, 3, 33, 256, 257, 512, 1025])
def test_table_layouts_match_the_library(M):
    m, n, is_sin, is_lo, valid = tc_image_layout(M)
    # sizes: CUDA-core tables padded to 256 B, then the image (b2d_dft_tables_bytes is host code: no GPU needed)
    assert (cc_table_floats(M) + m.size) * 4 == _lib.lib().b2d_dft_tables_bytes(M)
    mc, tc, sc = cc_table_layout(M)
    _, Nt, Ke, Ko = dft_dims(M)
    assert mc.size == 2 * (Ke + Ko) * Nt and mc.max() == M - 1 and sc.sum() == (Ke + Ko) * Nt
    rng = np.random.default_rng(M)
    for i in np.concatenate([np.arange(min(64, m.size)), rng.integers(0, m.size, 500), [m.size - 1]]):
        got = (int(m[i]), int(n[i]), bool(is_sin[i]), bool(is_lo[i]), bool(valid[i]))
        want = _decode(int(i), M)
        if not want[4]:
            assert not got[4], (i, got, want)
        else:
            assert got == want, (i, got, want)
    # every (bin, column, table) appears exactly once as hi and once as lo
    keys = m[valid] * (2 * Nt) + n[valid] * 2 + is_sin[valid]
    for part in (is_lo[valid], ~is_lo[valid]):
        assert np.unique(keys[part]).size == keys[part].size == 2 * M * Nt


def test_tf32_split():
    rng = np.random.default_rng(0)
    v = np.concatenate([rng.uniform(-1, 1, 10000), [0.0, 1.0, -1.0, 0.5 + 2 ** -12, 0.5 + 3 * 2 ** -12]])
    v = v.astype(np.float32)
    hi, lo = split_tf32(v)
    assert np.all(hi.view(np.uint32) & 0x1FFF == 0) and np.all(lo.view(np.uint32) & 0x1FFF == 0)
    assert np.all(np.abs(v.astype(np.float64) - hi) <= 2.0 ** -11 * np.abs(v))
    assert np.all(np.abs(v.astype(np.float64) - hi - lo) <= 2.0 ** -21 * np.abs(v))
    assert hi[-2] == np.float32(0.5) and hi[-1] == np.float32(0.5 + 2 ** -10)    # ties to even


def test_tensor_core_accumulation_budget():
    """3 wgmmas per chunk of 8 even bins, one ulp (2^-23) each: 48 steps at 256 bins (the count ir_build_tc.cu's
    accuracy note gives), 96 at 512, in place of the CUDA-core kernel's Ke rounded FMAs (2^-24 each)."""
    assert tc_accumulation_eps(256) == 48 * 2.0 ** -23 and tc_accumulation_eps(512) == 96 * 2.0 ** -23
    assert tc_accumulation_eps(2) == 3 * 2.0 ** -23 and tc_accumulation_eps(33) == 9 * 2.0 ** -23
    c = np.random.default_rng(3).normal(-2, 0.5, (2, 512)).astype(np.float32)
    _, b_cc = ir_reference(c, ops.IR_MAG_HANN)
    _, b_tc = ir_reference(c, ops.IR_MAG_HANN, tensor_cores=True)
    l1 = (np.exp(c.astype(np.float64)) / 128 * ir_weights(512)).sum(-1, keepdims=True)
    assert np.allclose(b_tc - b_cc, (tc_accumulation_eps(512) - 256 * 2.0 ** -24) * l1, rtol=1e-12)
