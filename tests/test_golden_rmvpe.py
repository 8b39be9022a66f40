"""The RMVPE goldens (tests/golden/make_golden_rmvpe.py, recorded from the live reference on the CPU) against the
package's parameter tree and the float64 oracle (tests/rmvpe_oracle.py), no GPU.  tests/test_gpu_rmvpe.py replays the
same files through the kernels."""
import json
import os

import numpy as np
import pytest
import torch

from ddsp_svc_b200 import rmvpe as R
from tests import rmvpe_oracle as ro
from tests.golden import make_golden_rmvpe as mk


def test_state_dict_trees_match_the_reference():
    with open(os.path.join(mk.HERE, "rmvpe_state_dicts.json")) as f:
        trees = json.load(f)
    args = {"full": (4, 1, (2, 2)), "reduced": (1, 1, (2, 2), 2, 1)}
    for name, tree in trees.items():
        ours = R.E2E0(*args[name]).state_dict()
        assert list(ours) == list(tree), name
        assert all(list(v.shape) == tree[k] for k, v in ours.items()), name


@pytest.mark.parametrize("name", list(mk.CASES))
def test_golden_is_unsaturated(name):
    d, _ = mk.load(name)
    h = d["hidden64"]
    assert ((h > 0.01) & (h < 0.99)).mean() >= 0.5


@pytest.mark.parametrize("name", list(mk.CASES))
def test_oracle_replays_golden(name):
    d, m = mk.load(name)
    with torch.no_grad():
        if "audio" in d:
            f0, hid = ro.infer(m, torch.from_numpy(d["audio"]).double()[None], int(d["sr"]))
        else:
            hid = ro.mel2hidden(m, torch.from_numpy(d["mel"]).double())
            f0 = ro.decode(hid)
    # from audio the two sides hold HTK bases built by different code (each within an fp32 ulp of librosa's)
    tol, rtol = (1e-6, 1e-7) if "audio" in d else (1e-9, 1e-12)
    assert np.abs(hid.numpy() - d["hidden64"]).max() < tol
    assert np.allclose(f0.numpy(), d["f0_64"], rtol=rtol, atol=0)
    if "hidden32" in d:         # the reference's own fp32 run on the CPU, for scale
        assert np.abs(d["hidden32"] - d["hidden64"]).max() < 1e-3
