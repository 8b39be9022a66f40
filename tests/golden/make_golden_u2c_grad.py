"""Generate tests/golden/u2c_grad_*.npz: the LIVE reference's own autograd gradients of Unit2Control with the
convolution-only decoder (ddsp/unit2control.py with ConformerNaiveEncoder(conv_only=True)) with respect to every
parameter, on the CPU, in fp32 and (module ``.double()``) in float64.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_u2c_grad.py [case names; default: all]

The reference class gets this package's seeded weights (``build_model``: the default initialisation with the norms'
weights and biases moved off 1 / 0) loaded strictly; the loss is ``(dense * cot_dense).sum() + (hidden * cot_hidden).sum()``
with seeded cotangents, either of which a case may leave out.  Parameter gradients of a real-width model are ~2.7 M
floats, so tensors of up to 1024 elements are stored whole and larger ones as a fixed seeded sample of 1024 entries
(``sample_index``) plus their Frobenius norm -- the scheme u2c_gpu_*.npz uses for outputs.  Per parameter ``p``:
``f32/p`` and ``f64/p`` (the stored entries of the fp32 and the float64 gradient), ``norm/p`` (Frobenius norm of the
float64 gradient) and ``err32/p`` (relative RMS of fp32 - float64 over the WHOLE tensor: the reference's own fp32 error,
which bounds the kernels' in tests/test_gpu_unit2control_backward.py); ``none`` lists the parameters whose gradient is
None.  The tests import ``CASES`` / ``build_model`` / ``build_inputs`` from here and only read the stored files.
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

HERE = os.path.dirname(os.path.abspath(__file__))
SUPERFAST = OrderedDict((k, 1025) for k in ("harmonic_magnitude", "harmonic_phase", "noise_magnitude", "noise_phase"))
SMALL = OrderedDict([("a", 33), ("b", 7)])

CASES = OrderedDict([
    # real width; T not a multiple of the 64-frame tile; a repeated speaker id; zero f0 frames; both cotangents
    ("u2c_grad_stack_spk3_aug", dict(n_unit=768, n_spk=3, splits=SUPERFAST, use_conv_stack=True, use_pitch_aug=True, B=3, T=150,
                                     spk=[2, 3, 2], aug=[2.0, -3.0, 0.5], cot=("dense", "hidden"))),
    ("u2c_grad_plain_spk1", dict(n_unit=64, n_spk=1, splits=SMALL, use_conv_stack=False, use_pitch_aug=False, B=2, T=70,
                                 cot=("dense",))),
    # T < 31: every frame sees the zero padding of the depthwise convolution on both sides; hidden cotangent only
    ("u2c_grad_short_t20", dict(n_unit=64, n_spk=3, splits=SMALL, use_conv_stack=True, use_pitch_aug=True, B=2, T=20,
                                spk=[1, 3], cot=("hidden",))),                           # pitch-aug model called without aug_shift
    ("u2c_grad_aug_t129", dict(n_unit=64, n_spk=2, splits=SMALL, use_conv_stack=False, use_pitch_aug=True, B=1, T=129,
                               spk=[2], aug=[-4.0], cot=("dense", "hidden"))),
])


def path(name):
    return os.path.join(HERE, name + ".npz")


def _seed(name):
    return 1000 + list(CASES).index(name)


def sample_index(n, seed, k=1024):
    """indices of the stored entries of a flattened gradient of n elements (all of them up to 1024)"""
    if n <= k:
        return torch.arange(n)
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:k].sort().values


def model_kwargs(name):
    c = CASES[name]
    return dict(input_channel=c["n_unit"], n_spk=c["n_spk"], output_splits=c["splits"], use_pitch_aug=c["use_pitch_aug"],
                use_conv_stack=c["use_conv_stack"])


def build_model(name):
    """this package's Unit2Control (convolution-only decoder) on the CPU with the case's seeded weights"""
    from ddsp_svc_b200.unit2control import Unit2Control
    torch.manual_seed(_seed(name))
    m = Unit2Control(use_naive_v2=True, **model_kwargs(name))
    g = torch.Generator().manual_seed(_seed(name) + 1)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.startswith("norm.") or n.startswith("stack.1."):
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


def gradients(module, inp, dtype):
    """parameter gradients {name: tensor or None} of ``module`` (the reference's class, the oracle's or this package's)
    under the case's loss; floating inputs are cast to ``dtype``"""
    cast = lambda t: t.to(dtype=dtype, device=next(module.parameters()).device) if t is not None else None
    dev = next(module.parameters()).device
    module.zero_grad(set_to_none=True)
    ctrls, hidden = module(cast(inp["units"]), cast(inp["f0"]), cast(inp["phase"]), cast(inp["volume"]),
                           spk_id=None if inp["spk_id"] is None else inp["spk_id"].to(dev), aug_shift=cast(inp["aug_shift"]))
    loss = 0
    if inp["cot_dense"] is not None:
        loss = loss + (torch.cat(list(ctrls.values()), -1) * cast(inp["cot_dense"])).sum()
    if inp["cot_hidden"] is not None:
        loss = loss + (hidden * cast(inp["cot_hidden"])).sum()
    loss.backward()
    return OrderedDict((n, None if p.grad is None else p.grad.detach().clone()) for n, p in module.named_parameters())


def stored(name, grads):
    """{parameter: the entries of its gradient that the golden keeps}"""
    return OrderedDict((n, g.reshape(-1).cpu()[sample_index(g.numel(), _seed(name) + 10 + i)])
                       for i, (n, g) in enumerate(grads.items()) if g is not None)


def run_reference(name):
    with contextlib.redirect_stdout(io.StringIO()):
        ref_loader.load()
    from ddsp.unit2control import Unit2Control as Ref
    ours, inp = build_model(name), build_inputs(name)
    out = {}
    for dtype in (torch.float32, torch.float64):
        ref = Ref(use_naive_v2=True, **model_kwargs(name)).train()
        ref.load_state_dict(ours.state_dict())
        out[dtype] = gradients(ref.to(dtype), inp, dtype)
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
