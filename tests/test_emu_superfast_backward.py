"""csrc/superfast.cu's BACKWARD kernel source executed on the CPU (tests/emu/host_emu.h) against the reference's
autograd gradients (tests/golden/superfast_grad_*.npz), race-checked under ThreadSanitizer, plus the argument checks
of its C ABI entry (no device touched).  The kernel itself runs on hardware in tests/test_gpu_superfast_backward.py."""
import ctypes

import numpy as np
import pytest

from ddsp_svc_b200 import _lib
from tests import util
from tests.emu_harness import abi_call, assert_race_free, shared, tsan
from tests.golden import make_golden_superfast_grad as GG
from tests.test_emu_superfast import frame_par
from tests import regimes as R

P, NB = GG.P, GG.WIN // 2 + 1
f32 = np.float32
# per-control relative RMS bounds: the emulated comb source limits the harmonic side (the forward's emulation gate,
# 2e-7 abs at a signal RMS of ~0.009, is ~2e-5 relative); the noise side involves no comb
BOUND = {"harmonic_magnitude": 3e-5, "harmonic_phase": 3e-5, "noise_magnitude": 1e-5, "noise_phase": 1e-5}


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_superfast_bwd.cpp", tmp_path_factory)
    fp = ctypes.POINTER(ctypes.c_float)

    def run(f0, dense, noise, g, hops=29, seed=0, utt_off=0):
        B, nF = f0.shape[0], f0.shape[1]
        par = frame_par(np.asarray(f0).reshape(B, nF))
        dense = np.ascontiguousarray(dense, f32)
        nz = None if noise is None else np.ascontiguousarray(noise, f32)
        g = np.ascontiguousarray(g, f32)
        out = np.full((B, nF, 4 * NB), np.nan, f32)
        ptr = lambda a, off=0: ctypes.cast(a.ctypes.data + 4 * off, fp)
        rc = lib.emu_superfast_bwd(ptr(par), ptr(dense, 0), ptr(dense, NB), ptr(dense, 2 * NB), ptr(dense, 3 * NB),
                                   dense.shape[2], ptr(nz) if nz is not None else None, seed, utt_off, ptr(g), B, nF,
                                   hops, ptr(out))
        assert rc == 0
        return out

    return run


@pytest.mark.parametrize("name", list(GG.CASES))
@pytest.mark.parametrize("hops", [29, 5])
def test_backward_kernel_source_matches_reference_gradient(emu, name, hops):
    inp = GG.build_inputs(name)
    gold = np.load(GG.path(name))["grad"].astype(np.float64)
    got = emu(inp["f0"].numpy(), inp["dense"].numpy(), inp["noise"].numpy(), inp["cot"].numpy(), hops=hops)
    assert np.isfinite(got).all()
    for i, key in enumerate(GG.split_map()):
        ref = gold[..., i * NB:(i + 1) * NB]
        e = util.rms(got[..., i * NB:(i + 1) * NB] - ref) / util.rms(ref)
        assert e <= BOUND[key], (name, hops, key, e)


def test_in_kernel_noise_rows_are_shard_invariant(emu):
    inp = GG.build_inputs("superfast_grad_b2_f24")
    f0, dense, g = inp["f0"].numpy(), inp["dense"].numpy(), inp["cot"].numpy()
    full = emu(f0, dense, None, g, seed=3)
    part = emu(f0[1:], dense[1:], None, g[1:], seed=3, utt_off=1)
    assert np.isfinite(full).all() and np.array_equal(full[1:], part)
    assert not np.array_equal(full, emu(f0, dense, None, g, seed=4))


def test_backward_kernel_source_has_no_shared_memory_race(tmp_path):
    assert_race_free(tsan("tsan_superfast_bwd.cpp", tmp_path))


def test_backward_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    ok = dict(workspace=16, c_hm=16, c_hp=16, c_nm=16, c_np=16, ctrl_stride=4100, noise_in=0, seed=0, utterance_offset=0,
              grad_signal=16, B=1, n_frames=4, block=512, win_length=2048, grad_ctrl=16, stream=0)
    call = lambda **kw: abi_call("b2d_superfast_synth_backward", dict(ok, **kw))
    assert call(workspace=0) == -1 and call(grad_signal=0) == -1 and call(grad_ctrl=0) == -1            # B2D_ERR_NULL
    assert call(c_np=0) == -1
    assert call(B=0) == -2 and call(n_frames=0) == -2 and call(ctrl_stride=1024) == -2                 # B2D_ERR_SHAPE
    assert call(win_length=1024, ctrl_stride=513) == -4 and call(block=256) == -4                      # UNSUPPORTED
    assert call(B=70000) == -4
    assert call(grad_signal=20) == -3 and call(grad_ctrl=20) == -3 and call(noise_in=20) == -3         # B2D_ERR_ALIGN
    assert call(workspace=8) == -3
    assert b"superfast_synth_backward" in L.b2d_last_error()


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
    inp = R.build("superfast", *case, with_cotangents=True)
    got = emu(inp["f0"].numpy(), inp["dense"].numpy(), inp["noise"].numpy(), inp["cot"].numpy())
    assert np.isfinite(got).all()
    got = dict(zip(R.SPLITS["superfast"], np.split(got, 4, axis=-1)))
    for k, e in R.grad_errors(got, R.port_grad(inp), R.truth_grad(inp)).items():
        bound = R.grad_bound(e, 2.0)
        assert (e["got"] <= bound).all(), (case, k, e["got"], bound)
