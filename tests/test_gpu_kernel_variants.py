"""The compiled variants that the dispatchers of b2d_ir_build, b2d_sins_bank and b2d_ltv_fir pick outside the default
configuration: every instantiation of the oscillator bank (one to eight bases, several harmonic groups, both control
load paths), every direct-form FIR instantiation (block sizes 256 ... 2048, one or two jobs, up to 2048 taps) and whole
Sins / CombSub forwards that reach them.  Each case compares with a float64 restatement built from oracle/closed_form.py
on seeded inputs, against a per-output error bound, and asserts that the kernel instantiation it targets actually ran.
The impulse-response builders have their own module (test_gpu_ir_tc.py), which uses the references defined here.

Error model.  Each output is a sum of terms evaluated in fp32 (or 3xTF32, which carries fp32 precision).  Its error is
bounded by HEADROOM * EPS * (the l1 norm of the terms summed into it):
  * impulse-response tap: sum_m |w_m H_m| over the weighted spectrum (w = 1/L at DC and Nyquist, 2/L elsewhere),
    plus a worst-case term for the accumulation over the bins (ir_accumulation_eps): saturated all-pass controls make
    the phase step nearly constant, so the partial sums grow coherently and the rounding errors need not cancel;
  * bank sample: sum_h a_h A_h (1 + 2 pi |x|), a_h = the anchor (1..16) harmonic h is built from: the double-angle
    chain multiplies the error of the anchor's sine by up to a_h, and the fp32 argument a_h * 2 pi x carries a relative
    rounding error;
  * FIR output: sum_tau |h| |x| over the support, with |h| the largest of the three neighbouring frames' taps (the
    kernels interpolate through differences of neighbouring impulse responses).
The numbers measured on the GPU go to tests/report.record next to their bounds.
"""
import contextlib
import re

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib, ops, synthetic as syn
from oracle import closed_form as cf
from tests import report, util

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 44100

EPS = 2.0 ** -22
# Rounding errors of an fp32 sum of K terms of random sign (the bank and FIR inputs here) grow like sqrt(K) * 2^-24 of
# its l1 norm; those sums have K <= 1025 terms per accumulator, and sqrt(1025) * 2^-24 = 8 * EPS.  The impulse-response
# taps, whose inputs are built to make the sums coherent, add a worst-case accumulation term (ir_accumulation_eps).
HEADROOM = 8.0


def ir_accumulation_eps(M, tensor_cores):
    """Relative error budget of the accumulation over the bins of an impulse-response tap: the CUDA-core kernel rounds
    each of its Ke = (M + 1) / 2 FMAs per accumulator to nearest (<= 2^-24 of the running sum, which never exceeds the
    l1 norm); the tensor-core kernel truncates (tc_accumulation_eps)."""
    return tc_accumulation_eps(M) if tensor_cores else (M + 1) // 2 * 2.0 ** -24


def tc_accumulation_eps(M):
    """Relative error budget of the wgmma accumulation in ir_build_tc.cu: its fp32 accumulators truncate, losing up to
    one ulp (<= 2^-23 of the running sum, whose magnitude never exceeds the l1 norm) per wgmma.  Truncation errors all
    lean the same way, so they add up linearly: 3 wgmmas (hi*hi, lo*hi, hi*lo) per chunk of 8 bins, ceil(Ke / 8) chunks
    per parity (Ke = (M + 1) / 2 even bins).  M = 512: 96 steps, 1.1e-5."""
    return 3 * (((M + 1) // 2 + 7) // 8) * 2.0 ** -23
# whole forwards: error RMS relative to the signal RMS, the ratio test_sins_forward_vs_float64_truth allows
# (1e-6 on a signal of about 8e-3 RMS)
E2E_REL_RMS = 1.25e-4


# ---------------------------------------------------------------------------------------------------------------------
# launch check
# ---------------------------------------------------------------------------------------------------------------------
_profiler_started = False


def _kernel_names(fn, *args, **kwargs):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn(*args, **kwargs)
        torch.cuda.synchronize()
    cuda = torch.autograd.DeviceType.CUDA
    return out, [e.name for e in prof.events() if getattr(e, "device_type", None) == cuda]


def profiled(fn, *args, **kwargs):
    """-> (fn(*args, **kwargs), demangled names of the CUDA kernels it launched), recorded by torch.profiler with CUDA
    activities only.  The first profiling session of a process starts CUPTI and comes back without kernel records, so
    one session around a trivial kernel runs first.  A later session occasionally comes back without kernel records as
    well, either empty or holding only the copies fn made; fn (a pure call here) is then run again under a fresh session,
    up to PROFILE_ATTEMPTS times in all."""
    global _profiler_started
    if not _profiler_started:
        _kernel_names(lambda: torch.ones(1, device=DEV).add_(1))
        _profiler_started = True
    for _ in range(PROFILE_ATTEMPTS):
        out, names = _kernel_names(fn, *args, **kwargs)
        if any(not n.startswith(("Memcpy", "Memset")) for n in names):
            break
    return out, names


PROFILE_ATTEMPTS = 4


def assert_launched(names, *kernels):
    """Each of ``kernels`` (a name with its template arguments, e.g. 'sins_bank_kernel<6, false>') was launched.
    Call it after the numerical checks: without kernel records (CUPTI unavailable) only this assertion is skipped."""
    if not names:
        pytest.skip("the profiler recorded no CUDA kernels in %d sessions (CUPTI unavailable): numerics checked, "
                    "%s not asserted" % (PROFILE_ATTEMPTS, ", ".join(kernels)))
    for k in kernels:
        pat = r"(^|[\s:])" + re.escape(k) + (r"\(" if "<" in k else r"[<(]")
        assert any(re.search(pat, n) for n in names), (k, sorted(set(names)))


@contextlib.contextmanager
def fir_impl(name):
    ops.set_fir_impl(name)
    try:
        yield
    finally:
        ops.set_fir_impl("auto")


# ---------------------------------------------------------------------------------------------------------------------
# float64 references (no GPU needed)
# ---------------------------------------------------------------------------------------------------------------------
def ir_weights(M):
    """inverse real DFT weights of the M bins: 1/L at DC and Nyquist, 2/L elsewhere (L = 2(M-1))"""
    L = 2 * (M - 1)
    w = np.full(M, 2.0 / L)
    w[0] = w[-1] = 1.0 / L
    return w


def allpass_phase_fp32(c):
    """The group-delay phase the kernels and the reference evaluate: fp32 pi*tanh(c), fp64 running sum, fp32 emit."""
    gd = (np.float32(np.pi) * np.tanh(np.asarray(c, np.float32))).astype(np.float32)
    return np.cumsum(gd.astype(np.float64), axis=-1).astype(np.float32)


def allpass_spectrum_fp32(c):
    """exp(j phi) in float64 on the fp32 phase of allpass_phase_fp32."""
    return np.exp(1j * allpass_phase_fp32(c).astype(np.float64))


def allpass_phase_bound(c):
    """Per bin, a bound of |allpass_phase_fp32(c) - cumsum(pi tanh c)| (float64 phase): half an fp32 ulp of the emitted
    value plus, per summed term, 2^-22 of |pi tanh c| (fp32 pi, tanh and product)."""
    phi = allpass_phase_fp32(c)
    g = np.pi * np.abs(np.tanh(np.asarray(c, np.float64)))
    return 0.5 * np.spacing(np.abs(phi)).astype(np.float64) + np.cumsum(g * 2.0 ** -22, axis=-1)


def dynamic_window_u(f0, M, sr=SR):
    """u = (tau - L/2) / hw of the dynamic window, hw = 1.5 sr / (f0 + 1e-3), with u := 0 where u > 1: [..., L].
    u is float64, but the u > 1 rule is decided on the fp32 quotient, which is what the reference (fp32 torch) and
    the kernels compute: at the tap where u is within an fp32 rounding of 1 the float64 quotient can land on the other
    side (f0 = 696.3148 Hz, n_mag 512: 95 / hw is exactly 1 in fp32), and the window jumps from 0 to 1 there."""
    L = 2 * (M - 1)
    f0 = np.asarray(f0, np.float32)
    idx = np.arange(L) - L // 2
    u = idx / (1.5 * sr / (f0.astype(np.float64) + 1e-3))
    hw32 = np.float32(1.5) * np.float32(sr) / (f0 + np.float32(1e-3))
    u32 = idx.astype(np.float32) / hw32
    return np.where(u32 > 1, 0.0, u)


def ir_reference(c, mode, f0=None, sr=SR, tensor_cores=False):
    """float64 impulse responses [..., L] of raw controls c [..., M] and the per-tap error bound [..., L] of the
    CUDA-core kernel, or of the tensor-core kernel when ``tensor_cores``: HEADROOM * EPS * l1 for the evaluation of
    the terms (activations, sine and cosine, window, the final additions), plus the accumulation budget."""
    c = np.asarray(c, np.float32)
    M = c.shape[-1]
    if mode == ops.IR_ALLPASS:
        spec = allpass_spectrum_fp32(c)
        h = cf.impulse_response(spec, "none")
    elif mode == ops.IR_MAG_HANN:
        spec = np.exp(c.astype(np.float64)) / 128.0
        h = cf.impulse_response(spec, "hann")
    else:
        # closed_form's dynamic window, with its u > 1 rule decided in fp32 (dynamic_window_u)
        spec = np.exp(c.astype(np.float64))
        u = dynamic_window_u(np.asarray(f0, np.float32).reshape(c.shape[:-1] + (1,)), M, sr)
        h = cf.impulse_response(spec, "none") * (0.5 * (1.0 + np.cos(np.pi * u)))
    l1 = (np.abs(spec) * ir_weights(M)).sum(-1, keepdims=True)
    bound = HEADROOM * EPS * l1 * np.ones_like(h)
    if mode == ops.IR_MAG_DYNAMIC:
        # the window's cosine takes pi*u, computed in fp32 from an fp32 half width: its error grows with |u|
        # (hundreds of taps beyond a half width of a few taps when f0 is near Nyquist)
        bound = bound * (1.0 + 0.5 * np.pi * np.abs(u))
    return h, bound + ir_accumulation_eps(M, tensor_cores) * l1


def bank_reference(f0, c_amp, P, sr=SR):
    """float64 oscillator bank [B, T] (on the fp32-rounded phase, like the reference) and its per-sample bound."""
    x32 = cf.phase_cycles(f0, sr, P).astype(np.float32).astype(np.float64)
    A = cf.harmonic_amplitudes(c_amp, f0, sr)
    out = cf.sinusoid_bank(x32, A, P)
    anchor = np.arange(A.shape[-1]) % 16 + 1.0
    l1 = cf.upsample((A * anchor).sum(-1, keepdims=True), P)[..., 0]
    return out, HEADROOM * EPS * l1 * (1.0 + 2.0 * np.pi * np.abs(x32))


def fir_reference(x, ir, P):
    """float64 time-varying FIR [B, T] of x [B, T] with ir [B, nF, L] and its per-sample bound."""
    x = np.asarray(x, np.float64)
    a = np.abs(np.asarray(ir, np.float64))
    env = np.maximum(a, np.maximum(np.concatenate([a[:, :1], a[:, :-1]], 1), np.concatenate([a[:, 1:], a[:, -1:]], 1)))
    return cf.ltv_fir(x, ir, P), HEADROOM * EPS * cf.ltv_fir(np.abs(x), env, P)


def tf32_rn(v):
    """round-to-nearest-even to tf32 (10 explicit mantissa bits), as split_tf32 in ir_build_tc.cu"""
    u = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    return (u & 0xFFFFFFFF).astype(np.uint32).view(np.float32)


def split_tf32(v):
    v = np.asarray(v, np.float32)
    hi = tf32_rn(v)
    return hi, tf32_rn(v - hi)


def dft_dims(M):
    """(L, Nt, Ke, Ko): taps, output columns t = 0..Nt-1, even and odd bins"""
    return 2 * (M - 1), (M - 1) // 2 + 1, (M + 1) // 2, M // 2


def dft_value(m, t, is_sin, M):
    """cos / sin(2 pi m t / L) in float64, reduced exactly"""
    L = 2 * (M - 1)
    ang = 2.0 * np.pi * ((np.asarray(m, np.int64) * np.asarray(t, np.int64)) % L) / L
    return np.where(is_sin, np.sin(ang), np.cos(ang))


def cc_table_layout(M):
    """(m, t, is_sin) of every float of the CUDA-core tables cosE [Ke][Nt] | cosO [Ko][Nt] | sinE [Ke][Nt] |
    sinO [Ko][Nt] (ir_build.cu), in memory order."""
    _, Nt, Ke, Ko = dft_dims(M)
    rows_m = np.concatenate([2 * np.arange(Ke), 2 * np.arange(Ko) + 1] * 2)
    rows_sin = np.repeat([False, True], Ke + Ko)
    return np.repeat(rows_m, Nt), np.tile(np.arange(Nt), len(rows_m)), np.repeat(rows_sin, Nt)


def cc_table_floats(M):
    """floats the CUDA-core tables occupy in the buffer, padded to 256 bytes"""
    _, Nt, Ke, Ko = dft_dims(M)
    return (2 * (Ke + Ko) * Nt * 4 + 255) // 256 * 64


def tc_image_layout(M):
    """(m, n, is_sin, is_lo, valid) of every float of the tensor-core operand image, in memory order
    [chunk of 8 k][cosE hi, cosE lo, sinE hi, sinE lo, cosO hi, cosO lo, sinO hi, sinO lo][2 halves of 4 k][Npad][4]
    with bin m = 2k (E) or 2k+1 (O) and column n (ir_build_tc.cu); entries past Nt or past the bins are zero."""
    _, Nt, Ke, Ko = dft_dims(M)
    Npad, NC = (Nt + 15) // 16 * 16, (Ke + 7) // 8
    ch, blk, half, n, e = np.meshgrid(np.arange(NC), np.arange(8), np.arange(2), np.arange(Npad), np.arange(4),
                                      indexing="ij")
    k = 8 * ch + 4 * half + e
    odd = blk >= 4
    m = 2 * k + odd
    valid = (n < Nt) & (k < np.where(odd, Ko, Ke))
    return tuple(a.reshape(-1) for a in (m, n, (blk >> 1) & 1 == 1, blk & 1 == 1, valid))


def cc_row_of(m, is_sin, M):
    """row of bin m in the CUDA-core tables"""
    _, _, Ke, Ko = dft_dims(M)
    m = np.asarray(m)
    return np.where(m % 2 == 0, m // 2, Ke + m // 2) + np.where(is_sin, Ke + Ko, 0)


def tc_image_from_values(M, cc_values):
    """the operand image the library should store, from the CUDA-core table values cc_values (fp32)"""
    _, Nt, _, _ = dft_dims(M)
    m, n, is_sin, is_lo, valid = tc_image_layout(M)
    v = np.zeros(m.shape, np.float32)
    v[valid] = cc_values[cc_row_of(m[valid], is_sin[valid], M) * Nt + n[valid]]
    hi, lo = split_tf32(v)
    return np.where(is_lo, lo, hi)


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a, np.float32)).to(DEV)


def _check(name, got, want, bound, **extra):
    """record max |err| and the worst err / bound ratio; every output within its bound"""
    err = np.abs(np.asarray(got, np.float64) - want)
    ratio = float((err / bound).max())
    report.record(name, max_err=float(err.max()), max_bound=float(bound.max()), worst_err_over_bound=ratio,
                  ref_rms=util.rms(want), **extra)
    assert np.all(err <= bound), (name, ratio, float(err.max()))


# ---------------------------------------------------------------------------------------------------------------------
# oscillator bank (sins_bank.cu)
# ---------------------------------------------------------------------------------------------------------------------
def _bank_kernel(H):
    return "sins_bank_kernel<8, true>" if H > 128 else "sins_bank_kernel<%d, false>" % ((H + 15) // 16)


# (H, control load path, block): every instantiation (NB = 1, 3, 5, 6, 7, 8; two and four groups), both load paths
# for each H that is a multiple of 4, and block sizes 256 / 512 / 1024 across them
BANK_CASES = [(16, "tma", 256), (16, "fallback", 512), (48, "tma", 1024), (48, "fallback", 256),
              (80, "tma", 512), (80, "fallback", 1024), (96, "tma", 256), (96, "fallback", 512),
              (112, "tma", 1024), (112, "fallback", 256), (128, "tma", 512), (128, "fallback", 1024),
              (129, "fallback", 256), (200, "tma", 512), (200, "fallback", 1024), (256, "tma", 256),
              (256, "fallback", 512), (512, "tma", 1024), (512, "fallback", 256)]


def _bank_controls(H, path, B, nF, g):
    """[B, nF, H] device view that can only take ``path``: the bulk-copy (TMA) path needs H % 4 == 0, a 16-byte aligned
    view and a frame stride % 4 == 0; the fallback view is offset by one float in rows of odd stride."""
    width = H + 8 if path == "tma" else H + 5
    dense = (torch.randn(B, nF, width, generator=g) * 0.5 - 2.0).to(DEV)
    c = dense[..., 4:4 + H] if path == "tma" else dense[..., 1:1 + H]
    tma = H % 4 == 0 and c.data_ptr() % 16 == 0 and c.stride(1) % 4 == 0
    assert tma == (path == "tma") and c.stride(0) == nF * c.stride(1)
    return c


def _bank_f0(H, B, nF, g):
    """f0 whose Nyquist cut-off harmonic moves through [0.4 H, 1.3 H] across the frames (up in one utterance, down in
    the other): the mask changes between neighbouring frames and the interpolation crosses it"""
    cut = np.linspace(0.4 * H, 1.3 * H, nF)
    f0 = np.stack([SR / 2 / cut, SR / 2 / cut[::-1]][:B]) * (1 + 0.01 * torch.rand(B, nF, generator=g).double().numpy())
    return torch.from_numpy(f0.astype(np.float32))[..., None]


@pytest.mark.parametrize("H,path,block", BANK_CASES)
def test_sins_bank_variant(H, path, block):
    g = torch.Generator().manual_seed(1000 + H + block)
    B, nF = 2, 10 if block < 1024 else 6
    f0 = _bank_f0(H, B, nF, g)
    c = _bank_controls(H, path, B, nF, g)
    want, bound = bank_reference(f0.numpy(), c.cpu().numpy(), block)
    f0d = f0.to(DEV)
    fp, _ = ops.phase_scan(f0d, block, SR)
    got, names = profiled(ops.sins_bank, f0d, fp, c, block, SR)
    _check("variants/bank_h%d_%s_p%d" % (H, path, block), got.cpu().numpy(), want, bound)
    assert_launched(names, _bank_kernel(H))


# ---------------------------------------------------------------------------------------------------------------------
# direct-form FIR (ltv_fir.cu)
# ---------------------------------------------------------------------------------------------------------------------
# (block, jobs, set_fir_impl, taps, instantiation): all five instantiations, tap counts across segment boundaries
FIR_CASES = [
    (256, 1, "cuda", 2, "ltv_fir_kernel<128, 6>"),
    (256, 2, "cuda", 514, "ltv_fir_kernel<128, 6>"),
    (768, 1, "cuda", 1026, "ltv_fir_kernel<128, 6>"),
    (512, 1, "cuda8", 512, "ltv_fir_kernel<128, 6>"),
    (512, 2, "cuda8", 1026, "ltv_fir_kernel<128, 6>"),
    (768, 2, "cuda", 510, "ltv_fir_kernel<256, 3>"),
    (1280, 1, "cuda", 2048, "ltv_fir_kernel<256, 3>"),
    (1024, 2, "cuda8", 1022, "ltv_fir_kernel<256, 3>"),
    (1280, 2, "cuda", 1024, "ltv_fir_kernel<512, 1>"),
    (2048, 2, "cuda8", 514, "ltv_fir_kernel<512, 1>"),
    (512, 1, "cuda", 2048, "ltv_fir16_kernel<64, 7>"),
    (512, 1, "cuda", 510, "ltv_fir16_kernel<64, 7>"),
    (512, 2, "cuda", 1024, "ltv_fir16_kernel<64, 7>"),
    (1024, 1, "cuda", 514, "ltv_fir16_kernel<64, 7>"),
    (1024, 2, "cuda", 2048, "ltv_fir16_kernel<256, 1>"),
    (2048, 1, "cuda", 1022, "ltv_fir16_kernel<256, 1>"),
    (2048, 2, "cuda", 2, "ltv_fir16_kernel<256, 1>"),
]


def in_kernel_noise(B, nF, P, seed, utterance_offset):
    """The library's in-kernel noise: a direct-form FIR whose impulse response is a unit impulse at tap L/2 passes its
    input through exactly (every frame has the same response, so the interpolation terms are zero)."""
    ir = torch.zeros(B, nF, 2, device=DEV)
    ir[..., 1] = 1.0
    with fir_impl("cuda"):
        return ops.ltv_fir(None, ir, P, seed=seed, utterance_offset=utterance_offset)


def fir_two_jobs(x1, ir1, x2, ir2, P, seed, utterance_offset):
    """b2d_ltv_fir with two jobs of equal tap count -> (y1, y2, mix); x = None draws in-kernel noise"""
    B, nF, L = ir1.shape
    y1, y2, mix = (torch.empty(B, nF * P, device=DEV) for _ in range(3))
    rc = _lib.lib().b2d_ltv_fir(ops._ptr(x1), ir1.data_ptr(), L, y1.data_ptr(), ops._ptr(x2), ir2.data_ptr(), L,
                                y2.data_ptr(), mix.data_ptr(), seed, utterance_offset, B, nF, P, ops._stream())
    _lib.check(rc, "b2d_ltv_fir")
    return y1, y2, mix


@pytest.mark.parametrize("block,jobs,impl,taps,kernel", FIR_CASES)
def test_direct_form_fir_variant(block, jobs, impl, taps, kernel):
    """One job: in-kernel noise through the filter.  Two jobs: an explicit signal and in-kernel noise, mixed as
    mix = y1 + y2.  Where the FFT-domain kernel also applies (block 512, <= 1024 taps) it must draw the same noise."""
    g = torch.Generator().manual_seed(block * 7 + taps + jobs)
    B, nF, seed, off = 2, 5, 4242 + taps, 3
    T = nF * block
    irs = [(torch.randn(B, nF, taps, generator=g) * 0.05).to(DEV) for _ in range(jobs)]
    noise = in_kernel_noise(B, nF, block, seed, off)
    name = "variants/fir_p%d_j%d_%s_l%d" % (block, jobs, impl, taps)
    x1 = (torch.rand(B, T, generator=g) * 2 - 1).to(DEV) if jobs == 2 else None
    with fir_impl(impl):
        if jobs == 1:
            y, names = profiled(ops.ltv_fir, None, irs[0], block, seed=seed, utterance_offset=off)
            outs = [y]
        else:
            outs, names = profiled(fir_two_jobs, x1, irs[0], None, irs[1], block, seed, off)
    inputs = [noise] if jobs == 1 else [x1, noise]
    refs = [fir_reference(x.cpu().numpy(), h.cpu().numpy(), block) for x, h in zip(inputs, irs)]
    for j, ((want, bound), got) in enumerate(zip(refs, outs)):
        _check(name + "/y%d" % (j + 1), got.cpu().numpy(), want, bound)
    if jobs == 2:
        assert torch.equal(outs[2], outs[0] + outs[1])        # mix = y1 + y2, summed in this order
        _check(name + "/mix", outs[2].cpu().numpy(), refs[0][0] + refs[1][0], refs[0][1] + refs[1][1])
    if block == 512 and taps <= 1024:
        with fir_impl("fft"):
            y_fft, fft_names = profiled(ops.ltv_fir, None, irs[-1], block, seed=seed, utterance_offset=off)
        _check(name + "/fft_same_noise", y_fft.cpu().numpy(), *refs[-1])
        assert_launched(fft_names, "ltv_fir_fft_kernel")
    assert_launched(names, kernel)


# ---------------------------------------------------------------------------------------------------------------------
# whole forwards outside the default configuration
# ---------------------------------------------------------------------------------------------------------------------
def _forward_inputs(B, nF, P, split_map, seed):
    f0 = syn.make_f0(B, nF, SR, P, seed=seed, sweep_row=1)
    dense, ctrls = syn.make_ctrl(B, nF, split_map, seed=seed + 1)
    noise = syn.uniform_noise(B, nF * P, seed + 2)
    return f0, dense, {k: v.numpy() for k, v in ctrls.items()}, noise


def _check_forward(name, outs, truth):
    rec = {}
    for key, got in zip(("signal", "harmonic", "noise"), outs):
        want = truth[key]
        rec[key + "_rel_rms"] = util.rms(got.cpu().numpy() - want) / util.rms(want)
    report.record(name, bound=E2E_REL_RMS, signal_rms=util.rms(truth["signal"]), **rec)
    for key, e in rec.items():
        assert e < E2E_REL_RMS, (name, key, e)


def _sins_forward(B, nF, P, H, Ma, Mn, seed):
    sm = syn.sins_split_map(H, Ma, Mn)
    f0, dense, ctrls, noise = _forward_inputs(B, nF, P, sm, seed)
    truth = cf.sins(f0.numpy(), ctrls, SR, P, noise.numpy())
    dc = syn.split_views(dense.to(DEV), sm)
    f0d = f0.to(DEV)
    fp, _ = ops.phase_scan(f0d, P, SR)
    outs, names = profiled(ops.sins_synth, f0d, fp, dc["amplitudes"], dc["group_delay"], dc["noise_magnitude"], P, SR,
                           noise_in=noise.to(DEV))
    return outs, truth, names


# block -> the direct-form instantiation that runs the two FIR jobs (harmonic all-pass + noise filter)
SINS_BLOCK_KERNELS = {256: "ltv_fir_kernel<128, 6>", 768: "ltv_fir_kernel<256, 3>", 1024: "ltv_fir16_kernel<256, 1>",
                      1280: "ltv_fir_kernel<512, 1>"}


@pytest.mark.parametrize("block", sorted(SINS_BLOCK_KERNELS))
def test_sins_forward_direct_form_blocks(block):
    outs, truth, names = _sins_forward(2, 6, block, 128, 256, 256, seed=50 + block)
    _check_forward("variants/sins_p%d" % block, outs, truth)
    assert_launched(names, SINS_BLOCK_KERNELS[block], "sins_bank_kernel<8, false>")


def test_sins_forward_multigroup_bank_and_cuda_core_irs():
    """H = 256 (two harmonic groups), all-pass n_mag 257 and noise n_mag 513 (both above the tensor-core limit), tap
    counts 512 / 1024: two FIR launches, the second adding the first's output."""
    outs, truth, names = _sins_forward(2, 8, 512, 256, 257, 513, seed=70)
    _check_forward("variants/sins_h256_m257_m513", outs, truth)
    assert_launched(names, "sins_bank_kernel<8, true>", "ir_build_kernel<0>", "ir_build_kernel<1>")
    assert sum("ltv_fir" in n for n in names) >= 2, sorted(set(names))


def test_combsub_forward_1025_bin_dynamic_window():
    """n_mag 256 / 1025 / 256: the dynamic-window impulse responses come from the CUDA-core kernel above 48 KB of
    shared memory, and their 2048 taps from the direct-form FIR (the FFT-domain kernel stops at 1024)."""
    B, nF, P = 2, 8, 512
    sm = syn.combsub_split_map(256, 1025, 256)
    f0, dense, ctrls, noise = _forward_inputs(B, nF, P, sm, seed=90)
    truth = cf.combsub(f0.numpy(), ctrls, SR, P, noise.numpy())
    dc = syn.split_views(dense.to(DEV), sm)
    f0d = f0.to(DEV)
    fp, _ = ops.phase_scan(f0d, P, SR)
    outs, names = profiled(ops.combsub_synth, f0d, fp, dc["group_delay"], dc["harmonic_magnitude"],
                           dc["noise_magnitude"], P, SR, noise_in=noise.to(DEV))
    _check_forward("variants/combsub_m1025", outs, truth)
    assert_launched(names, "ir_build_kernel<2>", "ltv_fir16_kernel<64, 7>")
