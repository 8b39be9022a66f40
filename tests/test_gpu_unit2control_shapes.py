"""Unit2Control on the GPU against a float64 evaluation of the same network, at the lengths inference produces:
T = 1 and 2 (a 0.1 s realtime block without context is about 9 frames), tile edges of the fused kernels (15, 31, 64,
65), a 5 s slice (430 frames at hop 512), the first length whose conv-1 input runs the TF32 split's grid-stride loop
(B T = 939 on 132 SMs) and a 60 s slice (5168), plus a batch of four utterances with their own speakers and pitch
shifts.  Every GEMM precision runs, with the fused linear attention on and off.

Reference: the restatement in tests/test_unit2control_host.py (this package's host logic with the kernels replaced by
their torch definitions, itself pinned to the reference class's goldens), run on the CPU as a second instance that
loads the GPU model's state dict.  In float64 it is the truth; in fp32 it measures what fp32 arithmetic itself costs on
the same case, which sets the scale of the bounds.

Error model and bounds (relative RMS over the controls and over the hidden output):
  * "fp32": cuBLAS SIMT GEMMs and the fused kernels (fp32, with fp64 GroupNorm statistics) are an fp32 evaluation in
    another summation order: at most 10x the fp32 restatement's own error on the same case (measured: up to 1.8x).
  * "3xtf32": the operands are fp32-grade (3xTF32 drops only the lo x lo term, 2^-24 relative), but the products are
    accumulated by the tensor cores, whose fp32 accumulators truncate instead of rounding to nearest
    (tests/test_gpu_kernel_variants.tc_accumulation_eps): the errors of a K-long dot product lean one way and add up
    linearly rather than as a random walk.  Bound 20x the fp32 restatement's error (measured: up to 9.6x, 1.8e-6 on
    the hidden output of the pcmer_norm / plain-conv variant, on an H100 SXM at 700 W).
  * "tf32": one TF32 pass per product (10-bit mantissas, 2^-11 relative per operand): 4e-4 on the controls, the figure
    ddsp_svc_b200/unit2control.py documents (3.4e-4 measured on an H100 SXM at 700 W); and at least 10x the fp32
    mode's error on the same case, which shows the precision switch reaches cuBLAS through torch's allow_tf32 flag.
    Except at one token (B T = 1): cuBLAS runs those products as matrix-vector kernels, which do not use TF32, and the
    error equals fp32's (measured)."""
import functools

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import unit2control as U
from tests import report, util
from tests import test_gpu_unit2control as G
from tests import test_unit2control_host as H

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VARIANTS = ["pcmer_sins", "naive_superfast", "pcmer_norm_plainconv"]
LENGTHS = [1, 2, 15, 31, 64, 65, 430, 939, 5168]
TF32_BOUND = 4e-4


class _Restatement(U.Unit2Control):
    """Unit2Control with the fused kernels replaced by their torch definitions and every product a plain addmm / matmul
    (tests/test_unit2control_host.py); runs on the CPU in the dtype of its parameters."""
    _layernorm = staticmethod(H._layernorm)
    _conv_module = H._conv_module
    _attention = H._attention
    forward = H._forward
    gemm_precision = "fp32"


@functools.lru_cache(maxsize=None)
def _weights(name, seed=3):
    kw, splits = G.VARIANTS[name]
    torch.manual_seed(seed)
    return U.Unit2Control(768, 3, splits, **kw).state_dict()


def _instance(cls, name, state):
    """a second instance + load_state_dict (deepcopy does not work on weight_norm)"""
    kw, splits = G.VARIANTS[name]
    m = cls(768, 3, splits, **kw)
    m.load_state_dict(state)
    return m.eval()


def _gpu_model(name, mode, fused=False, state=None):
    m = _instance(U.Unit2Control, name, _weights(name) if state is None else state).to(DEV)
    m.gemm_precision, m.fused_attention = mode, fused
    return m


@functools.lru_cache(maxsize=None)
def _shared_model(name):
    """one GPU instance per variant for the parametrized cases, which set its mode and fused_attention per case (so
    they also switch the packed weights back and forth)"""
    return _gpu_model(name, "3xtf32")


def _model(name, mode, fused):
    m = _shared_model(name)
    m.gemm_precision, m.fused_attention = mode, fused
    return m


def _calls(name, B):
    kw = G.VARIANTS[name][0]
    if B == 1:
        c = dict(spk_id=torch.LongTensor([[2]]))
        if kw.get("use_pitch_aug"):
            c["aug_shift"] = torch.tensor([[[-4.0]]])
        return [c]
    per_utt = dict(spk_id=torch.LongTensor([[1], [2], [3], [2]]))
    if kw.get("use_pitch_aug"):
        per_utt["aug_shift"] = torch.tensor([[[2.0]], [[-3.0]], [[0.5]], [[7.0]]])
    return [per_utt, dict(spk_id=torch.LongTensor([[1]]), spk_mix_dict={1: 0.25, 3: 0.75})]


def _dense(out):
    controls, hidden = out
    return torch.cat(list(controls.values()), -1).double().cpu().numpy(), hidden.double().cpu().numpy()


def _rel(got, want):
    return util.rms(got - want) / max(util.rms(want), 1e-30)


def _run(model, inputs, call, dtype, device):
    args = [t.to(device=device, dtype=dtype) for t in inputs]
    kw = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in call.items()}
    if "aug_shift" in kw:
        kw["aug_shift"] = kw["aug_shift"].to(dtype)
    with torch.no_grad():
        return _dense(model(*args, **kw))


@functools.lru_cache(maxsize=None)
def _reference(name, B, T, seed=3):
    """-> inputs, calls, [(float64 controls, float64 hidden, fp32 restatement's (controls, hidden) errors)] per call"""
    inputs = G._inputs(B, T, 768, 40 + T)
    calls = _calls(name, B)
    state = _weights(name, seed)
    r64 = _instance(_Restatement, name, state).double()
    r32 = _instance(_Restatement, name, state)
    refs = []
    for c in calls:
        c64, h64 = _run(r64, inputs, c, torch.float64, "cpu")
        c32, h32 = _run(r32, inputs, c, torch.float32, "cpu")
        refs.append((c64, h64, (_rel(c32, c64), _rel(h32, h64))))
    return inputs, calls, refs


def _errors(model, name, B, T, seed=3):
    inputs, calls, refs = _reference(name, B, T, seed)
    out = []
    for c, (c64, h64, e32) in zip(calls, refs):
        gc, gh = _run(model, inputs, c, torch.float32, DEV)
        out.append(((_rel(gc, c64), _rel(gh, h64)), e32))
    return out


def _cases():
    for name in VARIANTS:
        for T in LENGTHS:
            for fused in ([False, True] if name.startswith("pcmer") else [False]):
                yield name, 1, T, fused
        for fused in ([False, True] if name.startswith("pcmer") else [False]):
            yield name, 4, 200, fused


CASES = list(_cases())
IDS = ["%s-B%d-T%d%s" % (n, B, T, "-fused" if f else "") for n, B, T, f in CASES]


@pytest.mark.parametrize("mode", ["fp32", "3xtf32"])
@pytest.mark.parametrize("name,B,T,fused", CASES, ids=IDS)
def test_fp32_grade_modes_against_float64(name, B, T, fused, mode):
    factor = {"fp32": 10, "3xtf32": 20}[mode]
    model = _model(name, mode, fused)
    for i, ((e_c, e_h), (r_c, r_h)) in enumerate(_errors(model, name, B, T)):
        report.record("u2c_shapes/%s/%s/B=%d,T=%d,fused=%d/%d" % (name, mode, B, T, fused, i), controls_rel_rms=e_c,
                      hidden_rel_rms=e_h, fp32_restatement_controls=r_c, fp32_restatement_hidden=r_h,
                      controls_ratio=e_c / r_c, hidden_ratio=e_h / r_h)
        assert e_c <= factor * r_c and e_h <= factor * r_h, (i, e_c, r_c, e_h, r_h)


@pytest.mark.parametrize("name,B,T,fused", CASES, ids=IDS)
def test_tf32_mode_against_float64(name, B, T, fused):
    tf32 = _errors(_model(name, "tf32", fused), name, B, T)
    fp32 = _errors(_model(name, "fp32", fused), name, B, T)
    for i, (((e_c, e_h), _), ((f_c, f_h), _)) in enumerate(zip(tf32, fp32)):
        report.record("u2c_shapes/%s/tf32/B=%d,T=%d,fused=%d/%d" % (name, B, T, fused, i), controls_rel_rms=e_c,
                      hidden_rel_rms=e_h, fp32_mode_controls=f_c, bound=TF32_BOUND)
        assert e_c <= TF32_BOUND, (i, e_c)
        if B * T > 1:
            assert e_c >= 10 * f_c and e_h >= 10 * f_h, (i, e_c, f_c, e_h, f_h)


def test_switching_gemm_precision_gives_the_bits_of_a_fresh_instance():
    """The packed weights are keyed on the precision: one instance switched through every mode (and back) computes
    what a fresh instance in that mode computes, bit for bit.  (A variant without GroupNorm, whose fp64 atomics have no
    fixed order; the library GEMMs are deterministic for equal shapes on one device.)"""
    name, T = "pcmer_norm_plainconv", 150
    inputs, calls, _ = _reference(name, 1, T)
    switched = _gpu_model(name, "3xtf32")
    for mode in ("3xtf32", "fp32", "tf32", "3xtf32", "fp32"):
        switched.gemm_precision = mode
        got = _run(switched, inputs, calls[0], torch.float32, DEV)
        want = _run(_gpu_model(name, mode), inputs, calls[0], torch.float32, DEV)
        for a, b in zip(got, want):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), mode


@pytest.mark.parametrize("mode", ["3xtf32", "fp32"])
def test_load_state_dict_after_a_call_repacks(mode):
    """load_state_dict copies new values into the same parameter storage; the packed weights must follow (they are keyed
    on each parameter's storage and version counter).  After a call with the first weights, the output must match
    float64 of the second weights within the mode's bound, and be far from float64 of the first."""
    name, T = "pcmer_sins", 64
    factor = {"fp32": 10, "3xtf32": 20}[mode]
    model = _gpu_model(name, mode)
    ((first_c, _), (first_r, _)), = _errors(model, name, 1, T)
    assert first_c <= factor * first_r
    model.load_state_dict(_weights(name, seed=11))
    ((e_c, e_h), (r_c, r_h)), = _errors(model, name, 1, T, seed=11)
    ((o_c, _), _), = _errors(model, name, 1, T)
    report.record("u2c_shapes/reload/%s" % mode, controls_rel_rms=e_c, hidden_rel_rms=e_h, vs_old_weights=o_c)
    assert e_c <= factor * r_c and e_h <= factor * r_h
    assert o_c > 1e-2


def test_forward_restores_allow_tf32():
    """Every mode sets torch.backends.cuda.matmul.allow_tf32 for its own GEMMs only: the caller's setting is back after
    a forward, also after one that raises (CPU input before any GEMM; a bad spk_id after the first GEMMs)."""
    name, T = "pcmer_sins", 31
    inputs, calls, _ = _reference(name, 1, T)
    units, f0, phase, volume = (t.to(DEV) for t in inputs)
    prev = torch.backends.cuda.matmul.allow_tf32
    try:
        for setting in (False, True):
            for mode in ("3xtf32", "fp32", "tf32"):
                model = _gpu_model(name, mode)
                torch.backends.cuda.matmul.allow_tf32 = setting
                with torch.no_grad():
                    model(units, f0, phase, volume, spk_id=calls[0]["spk_id"].to(DEV))
                    assert torch.backends.cuda.matmul.allow_tf32 == setting, mode
                    with pytest.raises(ValueError):
                        model(units.cpu(), f0, phase, volume, spk_id=calls[0]["spk_id"].to(DEV))
                    assert torch.backends.cuda.matmul.allow_tf32 == setting, mode
                    with pytest.raises(ValueError):
                        model(units, f0, phase, volume, spk_id=torch.LongTensor([[1], [2]]).to(DEV))
                    assert torch.backends.cuda.matmul.allow_tf32 == setting, mode
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
