"""The oracle's restatement of Unit2Control with the convolution-only decoder (oracle/unit2control.py) reproduces the
reference's own autograd gradients (tests/golden/u2c_grad_*.npz, made from the reference's class on the CPU): float64 to
1e-12, fp32 bit for bit (the same torch layers applied in the same order).  That makes it the oracle for the full
parameter gradients and the large shapes of tests/test_gpu_unit2control_backward.py."""
import json

import numpy as np
import pytest
import torch

from oracle.unit2control import NaiveUnit2Control
from tests.golden import make_golden_u2c_grad as GG


def oracle_for(name, dtype):
    ours = GG.build_model(name)
    m = NaiveUnit2Control(**GG.model_kwargs(name)).train()
    m.load_state_dict(ours.state_dict())                       # strict: same keys and shapes as the package's module
    return m.to(dtype)


@pytest.mark.parametrize("name", list(GG.CASES))
def test_oracle_gradients_match_the_reference(name):
    gold = np.load(GG.path(name))
    none = set(json.loads(str(gold["none"])))
    for dtype, key in ((torch.float64, "f64/"), (torch.float32, "f32/")):
        grads = GG.gradients(oracle_for(name, dtype), GG.build_inputs(name), dtype)
        assert {n for n, g in grads.items() if g is None} == none
        for n, got in GG.stored(name, grads).items():
            want = gold[key + n]
            if dtype == torch.float32:
                assert np.array_equal(got.numpy(), want), n
            else:
                assert np.abs(got.numpy() - want).max() <= 1e-12 * max(float(gold["norm/" + n]), 1.0), n


def test_unused_layer_norms_and_absent_cotangents_leave_no_gradient():
    gold = np.load(GG.path("u2c_grad_short_t20"))
    none = set(json.loads(str(gold["none"])))
    assert {"decoder.encoder_layers.%d.norm.%s" % (i, p) for i in range(3) for p in ("weight", "bias")} <= none
    assert {"dense_out.bias", "dense_out.weight_g", "dense_out.weight_v", "aug_shift_embed.weight"} <= none   # hidden cotangent only
