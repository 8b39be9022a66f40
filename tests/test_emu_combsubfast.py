"""csrc/combsubfast.cu's KERNEL SOURCE executed on the CPU (tests/emu/host_emu.h: one std::thread per CUDA thread,
__syncthreads = barrier) against the live-reference goldens and the fp64 closed form.

This is what stands in for the GPU parity run of this kernel until it has executed on hardware: it exercises the real
index arithmetic, barrier placement, in-place pairing and overlap-add of the .cu file (fp32, like the device), for
full, ragged and single-frame chunks.  It cannot see PTX-level or performance problems."""
import ctypes

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import synthetic as syn
from oracle import closed_form as cf
from tests import util
from tests.golden import cases as G
from tests import regimes as R
from tests.emu_harness import shared

SR, P = G.SR, G.P


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_combsubfast.cpp", tmp_path_factory)
    fp = ctypes.POINTER(ctypes.c_float)

    def run(comb, dense, noise, G_hops=32, seed=0, utt_off=0):
        """comb [B,T] f32, dense controls [B,nF,3*(P+1)] f32 (views share the frame stride), noise [B,T] or None"""
        B, T = comb.shape
        nF = T // P
        comb = np.ascontiguousarray(comb, np.float32)
        dense = np.ascontiguousarray(dense, np.float32)
        out = np.full((B, T), np.nan, np.float32)
        ptr = lambda a, off=0: ctypes.cast(a.ctypes.data + 4 * off, fp)
        nz = None if noise is None else np.ascontiguousarray(noise, np.float32)
        rc = lib.emu_combsubfast(ptr(comb), ptr(dense, 0), ptr(dense, P + 1), ptr(dense, 2 * (P + 1)), dense.shape[2],
                                 ptr(nz) if nz is not None else None, seed, utt_off, B, nF, G_hops, ptr(out))
        assert rc == 0
        return out

    return run


def _comb_fp32(name_or_inputs):
    """the comb-tooth source as the reference computes it in fp32 (oracle port), [B, T]"""
    from oracle import torch_port as tp
    inp = name_or_inputs
    with torch.no_grad():
        x, f0_up = tp.wrapped_phase(inp["f0"], SR, P, inp.get("initial_phase"), True)
        return torch.sinc(torch.tensor(SR) * x / (f0_up + 1e-3)).squeeze(-1).numpy()


@pytest.mark.parametrize("name", [n for n, c in G.CASES.items() if c["kind"] == "combsubfast"])
@pytest.mark.parametrize("hops", [32, 16, 8, 4, 2])
def test_kernel_source_matches_reference_golden(emu, name, hops):
    inp = G.build_inputs(name)
    gold = util.load_golden(name)
    got = emu(_comb_fp32(inp), inp["dense"].numpy(), inp["noise"].numpy(), G_hops=hops)
    assert not np.isnan(got).any()
    e, m = util.rms(got - gold["signal"]), np.abs(got - gold["signal"]).max()
    assert e < 2e-7 and m < 2e-6, (name, hops, e, m)


def test_kernel_source_long_ragged_against_truth(emu):
    """70 frames = two full 32-hop chunks + a ragged chunk of 6; fp64 closed form as truth"""
    B, nF = 2, 70
    f0 = syn.make_f0(B, nF, SR, P, seed=5, unvoiced_fraction=0.2)
    dense, views = syn.make_ctrl(B, nF, syn.combsubfast_split_map(P), seed=6)
    noise = syn.uniform_noise(B, nF * P, 9)
    truth = cf.combsubfast(f0.numpy(), {k: v.numpy() for k, v in views.items()}, SR, P, noise.numpy())
    got = emu(_comb_fp32({"f0": f0}), dense.numpy(), noise.numpy())
    # bounds = the reference's own fp32 distance from the fp64 truth (tests/test_oracle_golden.py CF_BOUNDS)
    assert util.rms(got - truth["signal"]) < 5e-7
    assert np.abs(got - truth["signal"]).max() < 5e-6


def test_kernel_source_in_kernel_noise_is_shard_invariant(emu):
    B, nF = 3, 5
    f0 = syn.make_f0(B, nF, SR, P, seed=2)
    dense, _ = syn.make_ctrl(B, nF, syn.combsubfast_split_map(P), seed=3)
    comb = _comb_fp32({"f0": f0})
    full = emu(comb, dense.numpy(), None, seed=4)
    part = emu(comb[1:], dense.numpy()[1:], None, seed=4, utt_off=1)
    assert np.array_equal(full[1:], part) and np.isfinite(full).all()
    silent = emu(np.zeros_like(comb), dense.numpy(), None, seed=4)       # noise branch alone: non-trivial output
    assert 1e-4 < util.rms(silent) < 1.0


def test_output_is_bit_identical_for_any_chunking(emu):
    """frames are always transformed in the same (2m, 2m+1) pairs, so the hops-per-CTA choice (adapted to the batch size
    by the launcher) cannot change a single bit"""
    inp = G.build_inputs("csfast_b2_f24")
    comb, dense, noise = _comb_fp32(inp), inp["dense"].numpy(), inp["noise"].numpy()
    ref = emu(comb, dense, noise, G_hops=32)
    for hops in (2, 4, 8, 16):
        assert np.array_equal(emu(comb, dense, noise, G_hops=hops), ref), hops
    odd = emu(comb[:, :23 * P], dense[:, :23], noise[:, :23 * P], G_hops=32)       # odd frame count
    for hops in (2, 8):
        assert np.array_equal(emu(comb[:, :23 * P], dense[:, :23], noise[:, :23 * P], G_hops=hops), odd), hops


@pytest.mark.parametrize("case", R.TABLE, ids=R.CASE_IDS)
def test_kernel_source_at_input_regimes(emu, case):
    """The filter kernel source at the pitch and control regimes of tests/regimes.py (fed the reference's fp32 comb),
    to the criterion of tests/test_gpu_regimes_forward.py: within max(floor, 2 x the fp32 reference's own error) of
    float64, per row.
    The emulator evaluates __sinf, __sincosf, __expf and __fdividef with exact libm calls (tests/emu/host_emu.h), so
    this checks indexing, chunking and the host-visible arithmetic at these inputs; it says nothing about the SFU
    intrinsics' range reduction or large-argument error, which only tests/test_gpu_regimes_*.py see."""
    inp = R.build("combsubfast", *case)
    truth = R.truth_forward(inp)["signal"]
    with torch.no_grad():
        ref = R.port_forward(inp)["signal"].numpy()
    got = emu(_comb_fp32({"f0": inp["f0"]}), inp["dense"].numpy(), inp["noise"].numpy())
    assert np.isfinite(got).all()
    bad = R.within_budget(R.forward_errors(got, ref, truth), 2.0, 3.0)
    assert not bad, (case, bad)
