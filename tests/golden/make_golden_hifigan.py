"""Generate tests/golden/hifigan_*.npz: the LIVE reference's NSF-HiFiGAN Generator (nsf_hifigan/models.py:207-273) on
the CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT; oracle/ref_loader puts a matplotlib stand-in with ``use()`` in place
where matplotlib is missing, for nsf_hifigan/utils.py):

    python tests/golden/make_golden_hifigan.py [case names; default: all]

Weights are not stored: ``seeded_state_dict`` rebuilds them from a seed (tests/reflow_oracle.seeded_weights over the
reference's weight-normed parameters).  hifigan_state_dicts.json holds the key / shape tree of each model, with weight
norm attached and removed.  Each file holds the inputs ``x`` [B, 128, nF] and ``f0`` [B, nF], the source's draws in
the reference's order under ``torch.manual_seed(seed)`` -- ``rand_ini`` [1, 1, 9] with its first entry zeroed, then
``noise`` [B, nF upp, 9] = randn_like of the sines -- and the reference's fp32 output ``out32`` and ``out64``, the
module in float64 fed the same draws.  The noise is not stored (at B = 3, nF = 37 it alone is 2 MB of incompressible
floats): the file keeps its ``seed`` and a check of it (``noise_head``, the first frame's values, and ``noise_sum``, the
float64 sum), and ``draws`` regenerates it from torch's CPU generator and verifies it against that check.
"""
import json
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import hifigan_oracle, reflow_oracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
MODELS = OrderedDict([("small", dict(h=hifigan_oracle.SMALL, seed=41)), ("full", dict(h=hifigan_oracle.FULL, seed=42))])

CASES = OrderedDict([("hifigan_small_b%d_f%d" % (B, nF), dict(model="small", B=B, nF=nF))
                     for B in (1, 3) for nF in (1, 2, 37)])
CASES["hifigan_full_b1_f3"] = dict(model="full", B=1, nF=3)
CASES["hifigan_small_b2_f5_weightnorm"] = dict(model="small", B=2, nF=5, weight_norm=True)


def path(name):
    return os.path.join(HERE, name + ".npz")


def _seed(name):
    return 4000 + list(CASES).index(name)


def _reference():
    ref_loader.load()
    import nsf_hifigan.models as m
    return m


def seeded_state_dict(model):
    """the model's generator state dict with weight norm attached (weight_g / weight_v), every parameter seeded; built
    without the reference (the package's Generator has the same tree)"""
    import warnings
    from ddsp_svc_b200.hifigan import Generator
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen = Generator(hifigan_oracle.config(MODELS[model]["h"]))
    return reflow_oracle.seeded_weights(gen, MODELS[model]["seed"]).state_dict()


def draws(d):
    """(rand_ini [1, 1, 9], noise [B, nF upp, 9]) of a golden file ``d``, regenerated from its seed in the reference's
    order and checked against the stored head and sum of the noise the reference drew"""
    B = d["f0"].shape[0]
    g = torch.Generator().manual_seed(int(d["seed"]))
    rand_ini = torch.rand(1, 1, 9, generator=g)
    rand_ini[..., 0] = 0
    noise = torch.randn(B, d["out32"].shape[-1], 9, generator=g)
    if not (np.array_equal(rand_ini.numpy(), d["rand_ini"]) and np.array_equal(noise[0, :512].numpy(), d["noise_head"])
            and noise.double().sum().item() == float(d["noise_sum"])):
        raise AssertionError("the regenerated draws differ from the ones the reference made")
    return rand_ini, noise


def build_inputs(name):
    """x: a log-mel-like [B, 128, nF] (a ramp over the bins plus noise); f0 [B, nF]: 100-400 Hz with one unvoiced
    frame per utterance when nF > 1"""
    c = CASES[name]
    g = torch.Generator().manual_seed(_seed(name))
    B, nF = c["B"], c["nF"]
    x = torch.linspace(-8.0, 0.5, 128)[None, :, None] + 1.5 * torch.randn(B, 128, nF, generator=g)
    f0 = 100.0 + 300.0 * torch.rand(B, nF, generator=g)
    if nF > 1:
        f0[:, nF // 2] = 0.0
    return dict(x=x, f0=f0)


def generate(name):
    c = CASES[name]
    m = _reference()
    h = hifigan_oracle.config(MODELS[c["model"]]["h"])
    gen = m.Generator(h)
    gen.load_state_dict(seeded_state_dict(c["model"]), strict=True)
    if not c.get("weight_norm"):
        gen.remove_weight_norm()
    gen.eval()
    inp = build_inputs(name)
    out = {k: v.numpy() for k, v in inp.items()}
    B, nF = c["B"], c["nF"]
    with torch.no_grad():
        torch.manual_seed(_seed(name))
        out32 = gen(inp["x"], inp["f0"])
        torch.manual_seed(_seed(name))                      # the same draws, in the reference's order (models.py:144,163)
        rand_ini = torch.rand(1, 1, 9)
        rand_ini[..., 0] = 0
        noise = torch.randn(B, nF * gen.upp, 9)
        # replay with the draws substituted, in fp32 (must give out32 bit for bit) and in float64
        rand, randn_like = torch.rand, torch.randn_like
        torch.rand = lambda *a, **k: rand_ini.clone()
        torch.randn_like = lambda t, **k: noise.to(t.dtype)
        try:
            replay = gen(inp["x"], inp["f0"])
            out64 = gen.double()(inp["x"].double(), inp["f0"].double())
        finally:
            torch.rand, torch.randn_like = rand, randn_like
    assert torch.equal(replay, out32), "the substituted draws do not reproduce the reference's output"
    out.update(seed=np.int64(_seed(name)), rand_ini=rand_ini.numpy(), noise_head=noise[0, :512].numpy(),
               noise_sum=np.float64(noise.double().sum().item()), out32=out32.numpy(), out64=out64.numpy())
    np.savez_compressed(path(name), **out)
    r, n = draws(np.load(path(name)))
    assert torch.equal(r, rand_ini) and torch.equal(n, noise)


def write_state_dict_keys():
    """hifigan_state_dicts.json: [key, shape] of the reference's Generator for each model, with weight norm (as a
    checkpoint's 'generator' dict holds it) and after remove_weight_norm()"""
    m = _reference()
    sd = {}
    for model in MODELS:
        gen = m.Generator(hifigan_oracle.config(MODELS[model]["h"]))
        sd[model + "_weight_norm"] = [[k, list(v.shape)] for k, v in gen.state_dict().items()]
        gen.remove_weight_norm()
        sd[model] = [[k, list(v.shape)] for k, v in gen.state_dict().items()]
    with open(os.path.join(HERE, "hifigan_state_dicts.json"), "w") as f:
        json.dump(sd, f)


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    write_state_dict_keys()
    for n in names:
        generate(n)
        d = np.load(path(n))
        print("wrote", path(n), "out32 rms %.4f" % float(np.sqrt((d["out32"] ** 2).mean())),
              "|out32 - out64| max %.2e" % float(np.abs(d["out32"] - d["out64"]).max()))
