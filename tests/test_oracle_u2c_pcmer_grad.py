"""The oracle's restatement of Unit2Control with the PCmer decoder (tests/u2c_pcmer_oracle.py: PCmerUnit2Control)
reproduces the reference's own autograd gradients (tests/golden/u2c_pcmer_grad_*.npz, made from the reference's class on
the CPU): float64 to 1e-12, fp32 bit for bit (the same torch ops in the same order).  That makes it the oracle for the full
parameter gradients and the large shapes of tests/test_gpu_u2c_pcmer_backward.py.  Also the negative control for the
query features' row maximum: dropping its gradient moves query-side gradients by far more than the GPU tests' bounds."""
import json

import numpy as np
import pytest
import torch

from tests import util
from tests.golden import make_golden_u2c_pcmer_grad as GP
from tests.u2c_pcmer_oracle import PCmerUnit2Control


def oracle_for(name, dtype):
    ours = GP.build_model(name)
    m = PCmerUnit2Control(**GP.model_kwargs(name)).train()
    m.load_state_dict(ours.state_dict())                       # strict: same keys and shapes as the package's module
    return m.to(dtype)


@pytest.mark.parametrize("name", list(GP.CASES))
def test_oracle_gradients_match_the_reference(name):
    gold = np.load(GP.path(name))
    none = set(json.loads(str(gold["none"])))
    for dtype, key in ((torch.float64, "f64/"), (torch.float32, "f32/")):
        grads = GP.gradients(oracle_for(name, dtype), GP.build_inputs(name), dtype)
        assert {n for n, g in grads.items() if g is None} == none
        for n, got in GP.stored(name, grads).items():
            want = gold[key + n]
            if dtype == torch.float32:
                assert np.array_equal(got.numpy(), want), n
            else:
                assert np.abs(got.numpy() - want).max() <= 1e-12 * max(float(gold["norm/" + n]), 1.0), n


def test_every_pcmer_parameter_has_a_gradient_and_the_projection_is_a_buffer():
    gold = np.load(GP.path("u2c_pcmer_grad_sins_spk3"))
    assert json.loads(str(gold["none"])) == []
    keys = {k[4:] for k in gold.files if k.startswith("f64/")}
    for i in range(3):
        for p in ("norm.", "attn.to_q.", "attn.to_k.", "attn.to_v.", "attn.to_out.", "conformer.net.0.", "conformer.net.2.",
                  "conformer.net.4.conv.", "conformer.net.6."):
            assert {"decoder._layers.%d.%s%s" % (i, p, w) for w in ("weight", "bias")} <= keys
    assert not any("projection_matrix" in k for k in keys)
    short = set(json.loads(str(np.load(GP.path("u2c_pcmer_grad_short_t20"))["none"])))
    assert short == {"dense_out.bias", "dense_out.weight_g", "dense_out.weight_v"}      # hidden cotangent only


@pytest.mark.parametrize("name", ["u2c_pcmer_grad_sins_spk3", "u2c_pcmer_grad_norm_aug"])
def test_the_row_maximum_term_is_exercised(name):
    """float64: the oracle with the row maximum detached misses the term by more than 2e-5 relative RMS (the GPU tests'
    3xTF32 bound) on query-side tensors; the gradients of the key / value side and of everything after the attention stay"""
    gold, inp = np.load(GP.path(name)), GP.build_inputs(name)
    m = oracle_for(name, torch.float64)
    m.detach_max = True
    wrong = GP.stored(name, GP.gradients(m, inp, torch.float64))
    rel = {n: util.rms(g.numpy() - gold["f64/" + n]) / util.rms(gold["f64/" + n]) for n, g in wrong.items()}
    query = [n for n in rel if ".attn.to_q." in n]
    assert max(rel[n] for n in query) > 2e-5, rel
    assert all(rel[n] <= 1e-12 for n in rel if n.startswith("decoder._layers.2.conformer.") or n.startswith("dense_out."))
