"""csrc/ltv_fir_fft.cu's KERNEL SOURCE executed on the CPU (tests/emu/host_emu.h) against the oracle's time-varying
FIR (fp64 closed form of ddsp/core.py:120-182 and the bit-identical torch port), for one and two jobs, equal and
different tap counts, chunked / ragged hop ranges, the addend path and in-kernel noise."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import closed_form as cf
from tests import util
from tests import regimes as R
from tests.emu_harness import shared

P = 512


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_ltv_fir_fft.cpp", tmp_path_factory)
    fp = ctypes.POINTER(ctypes.c_float)

    def run(x1, ir1, x2=None, ir2=None, addend=None, hops=32, seed=0, utt_off=0, want=("y1", "y2", "mix")):
        B, nF, L1 = ir1.shape
        T = nF * P
        keep = []

        def ptr(a):
            if a is None:
                return None
            a = np.ascontiguousarray(a, np.float32)
            keep.append(a)
            return ctypes.cast(a.ctypes.data, fp)

        outs = {k: np.full((B, T), np.nan, np.float32) for k in want}
        optr = lambda k: ctypes.cast(outs[k].ctypes.data, fp) if k in outs else None
        L2 = ir2.shape[2] if ir2 is not None else 0
        rc = lib.emu_ltv_fir_fft(ptr(x1), ptr(ir1), L1, optr("y1"), ptr(x2), ptr(ir2), L2, optr("y2"), ptr(addend),
                                 optr("mix"), seed, utt_off, B, nF, hops)
        assert rc == 0
        return outs

    return run


def _case(B, nF, L, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, nF * P)).astype(np.float32)
    # smooth-ish random impulse responses that change from frame to frame
    ir = (rng.standard_normal((B, nF, L)) * np.hanning(L)[None, None, :] / np.sqrt(L)).astype(np.float32)
    return x, ir


@pytest.mark.parametrize("nF,hops", [(1, 32), (2, 32), (3, 32), (7, 4), (7, 2), (8, 2), (40, 32), (33, 32), (34, 32), (40, 16), (21, 8), (9, 4)])
def test_one_job_matches_closed_form(emu, nF, hops):
    x, ir = _case(2, nF, 510, nF)
    out = emu(x, ir, hops=hops, want=("y1", "mix"))
    truth = cf.ltv_fir(x.astype(np.float64), ir.astype(np.float64), P)
    assert not np.isnan(out["y1"]).any()
    scale = util.rms(truth)
    assert util.rms(out["y1"] - truth) < 2e-7 * max(scale, 1.0) and np.abs(out["y1"] - truth).max() < 5e-6
    assert np.array_equal(out["mix"], out["y1"])


@pytest.mark.parametrize("L1,L2", [(510, 510), (510, 254), (128, 512), (2, 2), (1022, 510), (514, 1024)])
def test_two_jobs_mix_and_addend(emu, L1, L2):
    nF = 9
    x1, ir1 = _case(2, nF, L1, 1)
    x2, ir2 = _case(2, nF, L2, 2)
    add = np.random.default_rng(3).standard_normal(x1.shape).astype(np.float32)
    out = emu(x1, ir1, x2, ir2, addend=add, hops=4)
    t1 = cf.ltv_fir(x1.astype(np.float64), ir1.astype(np.float64), P)
    t2 = cf.ltv_fir(x2.astype(np.float64), ir2.astype(np.float64), P)
    assert np.abs(out["y1"] - t1).max() < 5e-6 and np.abs(out["y2"] - t2).max() < 5e-6
    assert np.array_equal(out["mix"], (out["y1"] + out["y2"]) + add)          # same association as the direct kernel
    # outputs are optional
    only_mix = emu(x1, ir1, x2, ir2, hops=4, want=("mix",))
    assert np.array_equal(only_mix["mix"], out["y1"] + out["y2"])


def test_matches_the_reference_port_on_a_sins_like_case(emu):
    """impulse responses built like Sins' (all-pass + Hann-windowed noise filter), against the torch port that is
    bit-identical to the live reference"""
    from oracle import torch_port as tp
    torch.manual_seed(0)
    B, nF, M = 1, 12, 256
    gd = torch.pi * torch.tanh(torch.randn(B, nF, M) * 0.3)
    ir_ap = tp.impulse_response(torch.exp(1.j * torch.cumsum(gd, dim=-1)), "none")
    mag = torch.exp(torch.randn(B, nF, M) * 0.5 - 3.0) / 128
    ir_n = tp.impulse_response(torch.complex(mag, torch.zeros_like(mag)), "hann")
    x = torch.randn(B, nF * P) * 0.1
    z = torch.rand(B, nF * P) * 2 - 1
    ref_h, ref_n = tp.ltv_fir(x, ir_ap), tp.ltv_fir(z, ir_n)
    out = emu(x.numpy(), ir_ap.numpy(), z.numpy(), ir_n.numpy())
    # each channel to ITS OWN scale (the quiet noise channel must not inherit the harmonic channel's round-off)
    e_h, e_n = util.rms(out["y1"] - ref_h.numpy()), util.rms(out["y2"] - ref_n.numpy())
    assert e_h < 5e-7 * util.rms(ref_h.numpy()) + 1e-9, (e_h, util.rms(ref_h.numpy()))
    assert e_n < 5e-7 * util.rms(ref_n.numpy()) + 1e-9, (e_n, util.rms(ref_n.numpy()))
    assert util.rms(out["mix"] - (ref_h + ref_n).numpy()) < 1e-7


def test_in_kernel_noise_is_shard_invariant(emu):
    nF = 5
    x1, ir1 = _case(3, nF, 510, 4)
    _, ir2 = _case(3, nF, 510, 5)
    full = emu(x1, ir1, None, ir2, seed=7)
    part = emu(x1[1:], ir1[1:], None, ir2[1:], seed=7, utt_off=1)
    assert np.array_equal(full["y2"][1:], part["y2"]) and np.array_equal(full["mix"][1:], part["mix"])
    assert 1e-3 < util.rms(full["y2"]) < 10 and np.isfinite(full["mix"]).all()


@pytest.mark.parametrize("nF,hops,L", [(1, 32, 1022), (5, 2, 1022), (34, 32, 1022), (6, 32, 1024), (6, 4, 514)])
def test_one_job_long_filters_use_the_2048_point_transform(emu, nF, hops, L):
    """CombSub's 1022-tap harmonic filter: 512 + L - 1 > 1024, so the 2048-point instance runs"""
    x, ir = _case(2, nF, L, 10 + nF)
    out = emu(x, ir, hops=hops, want=("y1",))
    truth = cf.ltv_fir(x.astype(np.float64), ir.astype(np.float64), P)
    assert not np.isnan(out["y1"]).any()
    assert util.rms(out["y1"] - truth) < 2e-7 * max(util.rms(truth), 1.0) and np.abs(out["y1"] - truth).max() < 5e-6


def test_combsub_harmonic_filter_against_the_reference_port(emu):
    """dynamic-window 1022-tap impulse responses as CombSub builds them, against the port that is bit-identical to
    the live reference"""
    from oracle import torch_port as tp
    from tests.golden import cases as G
    name = "combsub_b2_f24"
    ref = util.port_outputs(name, G.build_inputs(name))
    out = emu(ref["allpassed"].numpy(), ref["ir_harmonic"].numpy(), want=("y1",))
    e = util.rms(out["y1"] - ref["harmonic"].numpy())
    assert e < 5e-7 * util.rms(ref["harmonic"].numpy()) + 1e-9, e


@pytest.mark.parametrize("L", [510, 1022])
def test_output_is_bit_identical_for_any_chunking(emu, L):
    """hops are always transformed in the same (2m, 2m+1) pairs, so the hops-per-CTA choice (which the launcher adapts to
    the batch size) and therefore batch splits / shards cannot change a single bit"""
    nF = 23
    x1, ir1 = _case(1, nF, L, 20)
    x2, ir2 = _case(1, nF, 510, 21)
    ref = emu(x1, ir1, x2, ir2, hops=32)
    for hops in (2, 4, 8, 16):
        out = emu(x1, ir1, x2, ir2, hops=hops)
        for k in ("y1", "y2", "mix"):
            assert np.array_equal(out[k], ref[k]), (hops, k)


def test_random_shapes_fuzz(emu):
    """25 random (batch, frames, hops per CTA, tap counts, one / two jobs, addend) combinations against the closed form"""
    rng = np.random.default_rng(123)
    for it in range(25):
        B, nF, hops = int(rng.integers(1, 3)), int(rng.integers(1, 12)), int(rng.choice([2, 4, 8, 16, 32]))
        L1 = int(rng.choice([2, 4, 64, 254, 510, 512, 514, 800, 1022, 1024]))
        two = bool(rng.integers(0, 2))
        L2 = int(rng.choice([2, 254, 510, 512, 1022]))
        x1 = rng.standard_normal((B, nF * P)).astype(np.float32)
        ir1 = (rng.standard_normal((B, nF, L1)) / np.sqrt(L1)).astype(np.float32)
        x2 = rng.standard_normal((B, nF * P)).astype(np.float32) if two else None
        ir2 = (rng.standard_normal((B, nF, L2)) / np.sqrt(L2)).astype(np.float32) if two else None
        add = rng.standard_normal((B, nF * P)).astype(np.float32) if rng.integers(0, 2) else None
        out = emu(x1, ir1, x2, ir2, addend=add, hops=hops, want=("y1", "y2", "mix") if two else ("y1", "mix"))
        tag = (it, B, nF, hops, L1, L2 if two else 0)
        assert np.abs(out["y1"] - cf.ltv_fir(x1.astype(np.float64), ir1.astype(np.float64), P)).max() < 1e-5, tag
        want = out["y1"]
        if two:
            assert np.abs(out["y2"] - cf.ltv_fir(x2.astype(np.float64), ir2.astype(np.float64), P)).max() < 1e-5, tag
            want = want + out["y2"]
        if add is not None:
            want = want + add
        assert np.array_equal(out["mix"], want), tag


# ---- spectrum path: ir_spectrum_kernel + the SPEC variant of the FIR kernel (impulse-response spectra read from memory) ----
@pytest.fixture(scope="module")
def emu_spec(tmp_path_factory):
    lib = shared("emu_ltv_fir_fft.cpp", tmp_path_factory)
    fp = ctypes.POINTER(ctypes.c_float)

    def run(x1, ir1, x2, ir2, hops=32, seed=0, utt_off=0):
        B, nF, L1 = ir1.shape
        T = nF * P
        keep = []

        def ptr(a):
            if a is None:
                return None
            a = np.ascontiguousarray(a, np.float32)
            keep.append(a)
            return ctypes.cast(a.ctypes.data, fp)

        outs = {k: np.full((B, T), np.nan, np.float32) for k in ("y1", "y2", "mix")}
        spec = [np.full((B, nF, 1024), np.nan, np.float32) for _ in range(2)]
        optr = lambda a: ctypes.cast(a.ctypes.data, fp)
        rc = lib.emu_ltv_fir_fft_spec(ptr(x1), ptr(ir1), L1, optr(outs["y1"]), ptr(x2), ptr(ir2), ir2.shape[2], optr(outs["y2"]),
                                      optr(outs["mix"]), seed, utt_off, B, nF, hops, optr(spec[0]), optr(spec[1]))
        assert rc == 0
        outs["spec1"], outs["spec2"] = spec
        return outs

    return run


@pytest.mark.parametrize("nF,hops,L1,L2", [(1, 32, 510, 510), (2, 2, 510, 510), (7, 4, 510, 254), (9, 2, 128, 512), (33, 32, 510, 510),
                                           (12, 8, 2, 510)])
def test_spectrum_path_matches_closed_form_and_packed_spectra(emu_spec, nF, hops, L1, L2):
    x1, ir1 = _case(2, nF, L1, 11)
    x2, ir2 = _case(2, nF, L2, 12)
    out = emu_spec(x1, ir1, x2, ir2, hops=hops)
    # the packed rows are the 1024-point spectra of the zero-padded taps: [0] = (DC, Nyquist), [k] = H[k]
    for ir, spec in ((ir1, out["spec1"]), (ir2, out["spec2"])):
        H = np.fft.rfft(ir.astype(np.float64), 1024, axis=-1)
        got = spec.reshape(*ir.shape[:2], 512, 2)
        assert np.abs(got[..., 0, 0] - H[..., 0].real).max() < 2e-6 and np.abs(got[..., 0, 1] - H[..., 512].real).max() < 2e-6
        assert np.abs((got[..., 1:, 0] + 1j * got[..., 1:, 1]) - H[..., 1:512]).max() < 2e-6
    t1 = cf.ltv_fir(x1.astype(np.float64), ir1.astype(np.float64), P)
    t2 = cf.ltv_fir(x2.astype(np.float64), ir2.astype(np.float64), P)
    assert not np.isnan(out["y1"]).any() and not np.isnan(out["mix"]).any()
    assert np.abs(out["y1"] - t1).max() < 5e-6 and np.abs(out["y2"] - t2).max() < 5e-6
    assert np.array_equal(out["mix"], out["y1"] + out["y2"])


def test_spectrum_path_is_bit_identical_for_any_chunking_and_shard(emu_spec):
    nF = 13
    x1, ir1 = _case(3, nF, 510, 21)
    _, ir2 = _case(3, nF, 510, 22)
    a = emu_spec(x1, ir1, None, ir2, hops=32, seed=5)
    b = emu_spec(x1, ir1, None, ir2, hops=2, seed=5)
    for k in ("y1", "y2", "mix"):
        assert np.array_equal(a[k], b[k]), k
    part = emu_spec(x1[1:], ir1[1:], None, ir2[1:], hops=4, seed=5, utt_off=1)
    assert np.array_equal(a["y2"][1:], part["y2"]) and np.array_equal(a["mix"][1:], part["mix"])


@pytest.mark.parametrize("synth,case", [("sins", ("octave_jumps", "saturated_gd")), ("sins", ("high", "phase_turns")),
                                        ("sins", ("onsets", "mixed_rows")), ("combsub", ("low", "trained")),
                                        ("combsub", ("glide", "hot")), ("combsub", ("near_zero", "cold"))],
                         ids=lambda v: v if isinstance(v, str) else "-".join(v))
def test_kernel_source_at_input_regimes(emu, synth, case):
    """The FFT-domain FIR kernel source on the filters of tests/regimes.py: Sins' saturated all-pass (510 taps) with the
    noise filter as second job, CombSub's dynamic-window harmonic filter (1022 taps), each fed the float64 stage before
    it rounded to fp32.  Within max(floor, 2 x the fp32 reference FIR's own error) of the float64 FIR, per row.
    The emulator evaluates __sinf, __sincosf, __expf and __fdividef with exact libm calls (tests/emu/host_emu.h), so
    this checks indexing, chunking and the host-visible arithmetic at these inputs; it says nothing about the SFU
    intrinsics' range reduction or large-argument error, which only tests/test_gpu_regimes_*.py see."""
    from oracle import torch_port as tp
    inp = R.build(synth, *case)
    t = R.truth_forward(inp)
    x1, ir1 = (t["sinusoids"], t["ir_allpass"]) if synth == "sins" else (t["allpassed"], t["ir_harmonic"])
    jobs = [(x1.astype(np.float32), ir1.astype(np.float32)), (inp["noise"].numpy(), t["ir_noise"].astype(np.float32))]
    out = emu(jobs[0][0], jobs[0][1], jobs[1][0], jobs[1][1], want=("y1", "y2"))
    for (x, ir), key in zip(jobs, ("y1", "y2")):
        truth = cf.ltv_fir(x, ir, P)
        ref = tp.ltv_fir(torch.from_numpy(x), torch.from_numpy(ir)).numpy()
        assert np.isfinite(out[key]).all()
        bad = R.within_budget(R.forward_errors(out[key], ref, truth), 2.0, 3.0)
        assert not bad, (synth, case, key, bad)
