"""csrc/combsubfast.cu's BACKWARD kernel source executed on the CPU (tests/emu/host_emu.h) against the reference's
autograd gradients (tests/golden/csfast_grad_*.npz), race-checked under ThreadSanitizer, plus the argument checks of
its C ABI entry (no device touched).  The kernel itself runs on hardware in tests/test_gpu_combsubfast_backward.py."""
import ctypes

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import _lib
from oracle import torch_port as tp
from tests import util
from tests.golden import make_golden_combsubfast_grad as GG
from tests import regimes as R
from tests.emu_harness import abi_call, assert_race_free, shared, tsan

P, NB = GG.P, GG.NB
f32 = np.float32
# per-control relative RMS bounds.  The emulation is fed the comb the reference filtered (the oracle port's, bit-identical),
# so both sides sit at the fp32 floor of 1.5 single-precision 1024-point transforms per frame
BOUND = {"harmonic_magnitude": 1e-5, "harmonic_phase": 1e-5, "noise_magnitude": 1e-5}


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_combsubfast_bwd.cpp", tmp_path_factory)
    fp = ctypes.POINTER(ctypes.c_float)

    def run(comb, dense, noise, g, hops=32, seed=0, utt_off=0):
        B, T = comb.shape
        nF = T // P
        comb = np.ascontiguousarray(comb, f32)
        dense = np.ascontiguousarray(dense, f32)
        nz = None if noise is None else np.ascontiguousarray(noise, f32)
        g = np.ascontiguousarray(g, f32)
        out = np.full((B, nF, 3 * NB), np.nan, f32)
        ptr = lambda a, off=0: ctypes.cast(a.ctypes.data + 4 * off, fp)
        rc = lib.emu_combsubfast_bwd(ptr(comb), ptr(dense, 0), ptr(dense, NB), ptr(dense, 2 * NB), dense.shape[2],
                                     ptr(nz) if nz is not None else None, seed, utt_off, ptr(g), B, nF, hops, ptr(out))
        assert rc == 0
        return out

    return run


def reference_comb(inp):
    """the comb the reference filters in the training phase (the oracle port's, bit-identical to it)"""
    with torch.no_grad():
        return tp.combsubfast_forward(inp["f0"], inp["ctrls"], GG.SR, P, noise=inp["noise"],
                                      initial_phase=inp["initial_phase"], infer=False)["comb"].numpy()


@pytest.mark.parametrize("name", list(GG.CASES))
@pytest.mark.parametrize("hops", [32, 2])
def test_backward_kernel_source_matches_reference_gradient(emu, name, hops):
    inp = GG.build_inputs(name)
    gold = np.load(GG.path(name))["grad"].astype(np.float64)
    got = emu(reference_comb(inp), inp["dense"].numpy(), inp["noise"].numpy(), inp["cot"].numpy(), hops=hops)
    assert np.isfinite(got).all()
    for i, key in enumerate(GG.split_map()):
        ref = gold[..., i * NB:(i + 1) * NB]
        e = util.rms(got[..., i * NB:(i + 1) * NB] - ref) / util.rms(ref)
        assert e <= BOUND[key], (name, hops, key, e)


def test_gradient_is_bit_identical_for_any_chunking(emu):
    """cotangent frames are always transformed in the same (2m, 2m+1) pairs and row nF-1 always adds frame nF to frame
    nF-1, so the rows-per-CTA choice cannot change a bit (odd and even frame counts)"""
    inp = GG.build_inputs("csfast_grad_b1_f70")
    comb, dense, noise, g = reference_comb(inp), inp["dense"].numpy(), inp["noise"].numpy(), inp["cot"].numpy()
    for nF in (70, 69):
        args = (comb[:, :nF * P], dense[:, :nF], noise[:, :nF * P], g[:, :nF * P])
        ref = emu(*args, hops=32)
        for hops in (2, 4, 16):
            assert np.array_equal(emu(*args, hops=hops), ref), (nF, hops)


def test_in_kernel_noise_rows_are_shard_invariant(emu):
    inp = GG.build_inputs("csfast_grad_b2_f24")
    comb, dense, g = reference_comb(inp), inp["dense"].numpy(), inp["cot"].numpy()
    full = emu(comb, dense, None, g, seed=3)
    part = emu(comb[1:], dense[1:], None, g[1:], seed=3, utt_off=1)
    assert np.isfinite(full).all() and np.array_equal(full[1:], part)
    other = emu(comb, dense, None, g, seed=4)
    # comb and noise share one complex transform: the harmonic side sees the other noise only through round-off
    harm, noise = np.s_[..., :2 * NB], np.s_[..., 2 * NB:]
    assert util.rms(full[harm] - other[harm]) <= 1e-5 * util.rms(full[harm])
    assert util.rms(full[noise] - other[noise]) >= 0.5 * util.rms(full[noise])


def test_backward_kernel_source_has_no_shared_memory_race(tmp_path):
    assert_race_free(tsan("tsan_combsubfast_bwd.cpp", tmp_path))


def test_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    ok = dict(comb=16, c_hm=16, c_hp=16, c_nm=16, ctrl_stride=3 * NB, noise_in=0, seed=0, utterance_offset=0,
              grad_signal=16, B=1, n_frames=4, block=512, grad_ctrl=16, stream=0)
    call = lambda **kw: abi_call("b2d_combsubfast_filter_backward", dict(ok, **kw))
    assert call(comb=0) == -1 and call(c_hm=0) == -1 and call(c_hp=0) == -1 and call(c_nm=0) == -1   # B2D_ERR_NULL
    assert call(grad_signal=0) == -1 and call(grad_ctrl=0) == -1
    assert call(B=0) == -2 and call(n_frames=0) == -2 and call(n_frames=-3) == -2                      # B2D_ERR_SHAPE
    assert call(ctrl_stride=512) == -2
    assert call(block=256) == -4 and call(block=1024) == -4 and call(B=70000) == -4                    # B2D_ERR_UNSUPPORTED
    assert call(comb=20) == -3 and call(grad_signal=20) == -3 and call(grad_ctrl=20) == -3             # B2D_ERR_ALIGN
    assert call(noise_in=20) == -3
    assert b"combsubfast_backward" in L.b2d_last_error()


@pytest.mark.parametrize("case", [("low", "saturated_gd"), ("high", "phase_turns"), ("onsets", "mixed_rows"),
                                  ("near_zero", "cold"), ("glide", "hot"), ("octave_jumps", "saturated_gd")],
                         ids=lambda c: "-".join(c))
def test_backward_kernel_source_at_input_regimes(emu, case):
    """The backward kernel source at the pitch and control regimes of tests/regimes.py, to the criterion of
    tests/test_gpu_regimes_backward.py: per control group and per row, relative L2 error against the float64 closed
    form within max(1e-5, 2 x the error of torch autograd through the fp32 port).
    The emulator evaluates __sinf, __sincosf, __expf and __fdividef with exact libm calls (tests/emu/host_emu.h), so
    this checks indexing, chunking and the host-visible arithmetic at these inputs; it says nothing about the SFU
    intrinsics' range reduction or large-argument error, which only tests/test_gpu_regimes_*.py see."""
    inp = R.build("combsubfast", *case, with_cotangents=True)
    got = emu(R.port_forward(inp, infer=False)["comb"].numpy(), inp["dense"].numpy(), inp["noise"].numpy(),
              inp["cot"].numpy())
    assert np.isfinite(got).all()
    got = dict(zip(R.SPLITS["combsubfast"], np.split(got, 3, axis=-1)))
    for k, e in R.grad_errors(got, R.port_grad(inp), R.truth_grad(inp)).items():
        bound = R.grad_bound(e, 2.0)
        assert (e["got"] <= bound).all(), (case, k, e["got"], bound)
