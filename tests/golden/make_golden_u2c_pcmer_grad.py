"""Generate tests/golden/u2c_pcmer_grad_*.npz: the LIVE reference's own autograd gradients of Unit2Control with the PCmer
decoder (ddsp/unit2control.py + ddsp/pcmer.py, training mode) with respect to every parameter, on the CPU, in fp32 and
(module ``.double()``) in float64.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_u2c_pcmer_grad.py [case names; default: all]

Same scheme as make_golden_u2c_grad.py (the convolution-only decoder's goldens): this package's seeded weights loaded
strictly into the reference's class, the loss ``(dense * cot_dense).sum() + (hidden * cot_hidden).sum()`` with seeded
cotangents, and per parameter ``p`` the fields ``f32/p``, ``f64/p`` (stored entries: whole tensors up to 1024 elements,
else a seeded sample of 1024), ``norm/p``, ``err32/p`` (the reference's own fp32 error, relative RMS over the whole
tensor) and ``none``.  ``ddsp.pcmer.FLAG_PCMER_NORM`` is process-global and a ``pcmer_norm=True`` constructor leaves it
set, so it is set explicitly for every case.  The tests import ``CASES`` / ``build_model`` / ``build_inputs`` /
``stored`` from here and only read the stored files.
"""
import contextlib
import io
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
from tests.golden.make_golden_u2c_grad import SMALL, gradients, sample_index  # noqa: E402,F401

HERE = os.path.dirname(os.path.abspath(__file__))
SINS = OrderedDict([("amplitudes", 128), ("group_delay", 256), ("noise_magnitude", 256)])       # configs/sins.yaml

CASES = OrderedDict([
    # real width, the Sins split map; T not a multiple of 64; a repeated speaker id; zero f0 frames; both cotangents
    ("u2c_pcmer_grad_sins_spk3", dict(n_unit=768, n_spk=3, splits=SINS, use_conv_stack=True, use_pitch_aug=False, pcmer_norm=False,
                                      B=3, T=150, spk=[2, 3, 2], cot=("dense", "hidden"))),
    # pcmer_norm (diffusion-new-fp16.yaml), plain first convolution, pitch augmentation with aug_shift
    ("u2c_pcmer_grad_norm_aug", dict(n_unit=64, n_spk=2, splits=SMALL, use_conv_stack=False, use_pitch_aug=True, pcmer_norm=True,
                                     B=2, T=70, spk=[2, 1], aug=[2.0, -3.0], cot=("dense",))),
    # T < 31: the depthwise convolution's padding on both sides of every frame; hidden cotangent only
    ("u2c_pcmer_grad_short_t20", dict(n_unit=64, n_spk=3, splits=SMALL, use_conv_stack=True, use_pitch_aug=False, pcmer_norm=False,
                                      B=2, T=20, spk=[1, 3], cot=("hidden",))),
    # one utterance, ragged length
    ("u2c_pcmer_grad_b1_t129", dict(n_unit=64, n_spk=1, splits=SMALL, use_conv_stack=True, use_pitch_aug=False, pcmer_norm=False,
                                    B=1, T=129, cot=("dense", "hidden"))),
])


def path(name):
    return os.path.join(HERE, name + ".npz")


def _seed(name):
    return 2000 + list(CASES).index(name)


def model_kwargs(name):
    c = CASES[name]
    return dict(input_channel=c["n_unit"], n_spk=c["n_spk"], output_splits=c["splits"], use_pitch_aug=c["use_pitch_aug"],
                pcmer_norm=c["pcmer_norm"], use_conv_stack=c["use_conv_stack"])


def build_model(name):
    """this package's Unit2Control (PCmer decoder) on the CPU with the case's seeded weights; every LayerNorm /
    GroupNorm weight and bias moved off 1 / 0"""
    from ddsp_svc_b200.unit2control import Unit2Control
    torch.manual_seed(_seed(name))
    m = Unit2Control(**model_kwargs(name))
    g = torch.Generator().manual_seed(_seed(name) + 1)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.startswith("norm.") or n.startswith("stack.1.") or ".norm." in n or ".net.0." in n:
                p.add_(0.2 * torch.randn(p.shape, generator=g))
    return m


def build_inputs(name):
    """units, f0 (with zero frames), phase, volume, spk_id / aug_shift (or None) and the two cotangents (or None)"""
    c = CASES[name]
    B, T = c["B"], c["T"]
    g = torch.Generator().manual_seed(_seed(name) + 2)
    units = torch.randn(B, T, c["n_unit"], generator=g)
    f0 = 220.0 * 2 ** (torch.rand(B, T, 1, generator=g) * 2 - 1)
    f0[:, 5:9] = 0.0
    phase = (torch.rand(B, T, 1, generator=g) * 2 - 1) * 3.14159
    volume = 0.2 * torch.rand(B, T, 1, generator=g)
    n_out = sum(c["splits"].values())
    cot_dense, cot_hidden = torch.randn(B, T, n_out, generator=g), torch.randn(B, T, 256, generator=g)
    return {"units": units, "f0": f0, "phase": phase, "volume": volume,
            "spk_id": torch.LongTensor(c["spk"]).reshape(B, 1) if "spk" in c else None,
            "aug_shift": torch.tensor(c["aug"]).reshape(B, 1, 1) if "aug" in c else None,
            "cot_dense": cot_dense if "dense" in c["cot"] else None, "cot_hidden": cot_hidden if "hidden" in c["cot"] else None}


def stored(name, grads):
    """{parameter: the entries of its gradient that the golden keeps}"""
    return OrderedDict((n, g.reshape(-1).cpu()[sample_index(g.numel(), _seed(name) + 10 + i)])
                       for i, (n, g) in enumerate(grads.items()) if g is not None)


def run_reference(name):
    with contextlib.redirect_stdout(io.StringIO()):
        ref_loader.load()
    from ddsp.unit2control import Unit2Control as Ref
    import ddsp.pcmer as ref_pcmer
    ours, inp = build_model(name), build_inputs(name)
    out = {}
    for dtype in (torch.float32, torch.float64):
        ref_pcmer.FLAG_PCMER_NORM = False
        ref = Ref(use_naive_v2=False, **model_kwargs(name)).train()
        ref_pcmer.FLAG_PCMER_NORM = CASES[name]["pcmer_norm"]
        ref.load_state_dict(ours.state_dict())
        out[dtype] = gradients(ref.to(dtype), inp, dtype)
    ref_pcmer.FLAG_PCMER_NORM = False
    return out[torch.float32], out[torch.float64]


def main():
    if not ref_loader.available():
        raise SystemExit("live reference not found; set DDSP_REFERENCE_ROOT to a DDSP-SVC checkout")
    for name in sys.argv[1:] or CASES:
        g32, g64 = run_reference(name)
        payload = {"none": np.array(json.dumps([n for n, g in g64.items() if g is None])),
                   "torch_version": np.array(torch.__version__)}
        for n, v in stored(name, g32).items():
            payload["f32/" + n] = v.numpy().astype(np.float32)
        for n, v in stored(name, g64).items():
            payload["f64/" + n] = v.numpy().astype(np.float64)
            payload["norm/" + n] = np.float64(g64[n].norm())
            payload["err32/" + n] = np.float64((g32[n].double() - g64[n]).norm() / g64[n].norm().clamp_min(1e-300))
        np.savez_compressed(path(name), **payload)
        print("%-28s %d gradients, %d None, %.0f kB" % (name, sum(k.startswith("f64/") for k in payload),
                                                         len(json.loads(str(payload["none"]))), os.path.getsize(path(name)) / 1e3))


if __name__ == "__main__":
    main()
