"""csrc/superfast.cu's main KERNEL SOURCE executed on the CPU (tests/emu/host_emu.h) against the live-reference
goldens.  The kernel is validated on hardware (tests/test_gpu_superfast.py); the emulation exists so that changes to
the shared FFT code can be checked -- and race-checked under ThreadSanitizer -- without a GPU.  The frame scan (warp
shuffles) is restated here in numpy with the kernel's fp32 operation order."""
import ctypes

import numpy as np
import pytest

from tests import util
from tests.golden import cases as G
import torch
from tests import regimes as R
from tests.emu_harness import shared

SR, P, WIN = G.SR, G.P, 2048
f32 = np.float32


def frame_par(f0):
    """(s, ds, acc_prev, 0) per frame as superfast_scan_kernel computes them (fp32 steps, fp64 running sum)"""
    f0 = np.asarray(f0, f32)
    B, nF = f0.shape
    s = (f0 / f32(SR)).astype(f32)
    ds = np.zeros_like(s)
    ds[:, :-1] = s[:, 1:] - s[:, :-1]
    fP, fPm1 = f32(P), f32(P - 1)
    t2 = (((f32(0.5) * ds).astype(f32) * fPm1).astype(f32) * fP).astype(f32)
    last = ((s * fP).astype(f32) + (t2 / fP).astype(f32)).astype(f32)
    adv = (np.fmod((last + f32(0.5)).astype(f32), f32(1.0)) - f32(0.5)).astype(f32)
    run = np.concatenate([np.zeros((B, 1)), np.cumsum(adv.astype(np.float64), axis=1)[:, :-1]], axis=1)
    accp = np.fmod(run.astype(f32), f32(1.0)).astype(f32)
    accp[:, 0] = 0
    return np.ascontiguousarray(np.stack([s, ds, accp, np.zeros_like(s)], axis=-1), f32)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_superfast.cpp", tmp_path_factory)
    fp = ctypes.POINTER(ctypes.c_float)

    def run(f0, dense, noise, hops=29, seed=0, utt_off=0):
        B, nF = f0.shape[0], f0.shape[1]
        par = frame_par(np.asarray(f0).reshape(B, nF))
        dense = np.ascontiguousarray(dense, f32)
        nz = None if noise is None else np.ascontiguousarray(noise, f32)
        out = np.full((B, nF * P), np.nan, f32)
        n = WIN // 2 + 1
        ptr = lambda a, off=0: ctypes.cast(a.ctypes.data + 4 * off, fp)
        rc = lib.emu_superfast(ptr(par), ptr(dense, 0), ptr(dense, n), ptr(dense, 2 * n), ptr(dense, 3 * n),
                               dense.shape[2], ptr(nz) if nz is not None else None, seed, utt_off, B, nF, hops, ptr(out))
        assert rc == 0
        return out

    return run


@pytest.mark.parametrize("name", [n for n, c in G.CASES.items() if c["kind"] == "superfast"])
@pytest.mark.parametrize("hops", [29, 5])
def test_kernel_source_matches_reference_golden(emu, name, hops):
    inp = G.build_inputs(name)
    gold = util.load_golden(name)
    got = emu(inp["f0"].numpy(), inp["dense"].numpy(), inp["noise"].numpy(), hops=hops)
    assert not np.isnan(got).any()
    e, m = util.rms(got - gold["signal"]), np.abs(got - gold["signal"]).max()
    assert e < 2e-7 and m < 5e-6, (name, hops, e, m)


def test_in_kernel_noise_is_shard_invariant(emu):
    inp = G.build_inputs("superfast_b2_f24")
    f0, dense = inp["f0"].numpy(), inp["dense"].numpy()
    full = emu(f0, dense, None, seed=3)
    part = emu(f0[1:], dense[1:], None, seed=3, utt_off=1)
    assert np.array_equal(full[1:], part) and np.isfinite(full).all()


@pytest.mark.parametrize("case", R.TABLE, ids=R.CASE_IDS)
def test_kernel_source_at_input_regimes(emu, case):
    """The forward kernel source at the pitch and control regimes of tests/regimes.py, to the criterion of
    tests/test_gpu_regimes_forward.py: within max(floor, 2 x the fp32 reference's own error) of float64, per row.
    The emulator evaluates __sinf, __sincosf, __expf and __fdividef with exact libm calls (tests/emu/host_emu.h), so
    this checks indexing, chunking and the host-visible arithmetic at these inputs; it says nothing about the SFU
    intrinsics' range reduction or large-argument error, which only tests/test_gpu_regimes_*.py see."""
    inp = R.build("superfast", *case)
    truth = R.truth_forward(inp)["signal"]
    with torch.no_grad():
        ref = R.port_forward(inp)["signal"].numpy()
    got = emu(inp["f0"].numpy(), inp["dense"].numpy(), inp["noise"].numpy())
    assert np.isfinite(got).all()
    bad = R.within_budget(R.forward_errors(got, ref, truth), 2.0, 3.0)
    assert not bad, (case, bad)
