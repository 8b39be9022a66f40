"""Generate tests/golden/sins_grad_*.npz: the LIVE reference's own autograd gradient of Sins (training phase,
infer=False) with respect to its three raw controls, on CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_sins_grad.py [case names; default: all]

The reference's Unit2Control is replaced by a module returning views of one leaf ``dense`` tensor that requires grad
(the split_to_dict layout, ddsp/unit2control.py:12-23); the noise is pinned by torch.manual_seed(seed) right before
forward(), as make_golden.py does; then ``(signal * cot + harmonic * cot_h + noise * cot_n).sum().backward()`` with
seeded cotangents (cot_h / cot_n only where the case says so).  Each .npz stores dense.grad [B, nF, H + Ma + Mn], the
signal, and float64 checksums of every input.

The case list lives here; the tests import ``CASES`` / ``build_inputs`` from this module and only read the stored files.
"""
import contextlib
import io
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from ddsp_svc_b200 import synthetic as syn  # noqa: E402
from oracle import ref_loader  # noqa: E402
from tests.golden import cases as G  # noqa: E402

SR, P = G.SR, G.P

CASES = OrderedDict([
    # configs/sins.yaml shape; unvoiced frames and a 65 -> 1100 Hz sweep row (harmonics cross Nyquist: the 1e-7 mask)
    ("sins_grad_b2_f24_h128", dict(B=2, nF=24, H=128, Ma=256, Mn=256, unvoiced=0.1, sweep_row=1)),
    # Ma != Mn, 200 harmonics (two harmonic groups, not a multiple of 32)
    ("sins_grad_b1_f5_h200_ma65_mn129", dict(B=1, nF=5, H=200, Ma=65, Mn=129)),
    ("sins_grad_b1_f1_h64", dict(B=1, nF=1, H=64, Ma=256, Mn=256)),
    ("sins_grad_b1_f2_h33", dict(B=1, nF=2, H=33, Ma=256, Mn=256)),
    ("sins_grad_b1_f4_h16_ma2_mn3", dict(B=1, nF=4, H=16, Ma=2, Mn=3)),
    # cotangents on harmonic and noise as well as on signal
    ("sins_grad_b2_f6_h128_parts", dict(B=2, nF=6, H=128, Ma=256, Mn=256, parts=True)),
])


def path(name):
    return os.path.join(G.HERE, name + ".npz")


def split_map(name):
    c = CASES[name]
    return syn.sins_split_map(c["H"], c["Ma"], c["Mn"])


def build_inputs(name):
    """f0 [B, nF, 1], dense raw controls + split views, U(-1, 1) noise [B, T], cotangents [B, T] (cot_h / cot_n None
    unless the case has parts)."""
    case = CASES[name]
    sd = G.seeds(name)
    B, nF = case["B"], case["nF"]
    f0 = syn.make_f0(B, nF, SR, P, seed=sd["f0"], unvoiced_fraction=case.get("unvoiced", 0.0),
                     sweep_row=case.get("sweep_row"))
    dense, views = syn.make_ctrl(B, nF, split_map(name), seed=sd["ctrl"])
    noise = syn.uniform_noise(B, nF * P, sd["noise"])
    g = torch.Generator().manual_seed(sd["noise"] + 1000)
    cot = torch.randn(B, nF * P, generator=g)
    cot_h = torch.randn(B, nF * P, generator=g) if case.get("parts") else None
    cot_n = torch.randn(B, nF * P, generator=g) if case.get("parts") else None
    return {"case": case, "f0": f0, "dense": dense, "ctrls": views, "noise": noise, "cot": cot, "cot_h": cot_h,
            "cot_n": cot_n}


def objective(signal, harmonic, noise, inp):
    out = (signal * inp["cot"]).sum()
    if inp["cot_h"] is not None:
        out = out + (harmonic * inp["cot_h"]).sum() + (noise * inp["cot_n"]).sum()
    return out


def input_checksums(inp):
    """cases.input_checksums (f0, dense, noise) plus the same checksum of each cotangent"""
    cs = G.input_checksums(inp)
    for k in ("cot", "cot_h", "cot_n"):
        if inp[k] is not None:
            t = inp[k].double()
            cs["cs_" + k] = float((t * torch.arange(1, t.numel() + 1, dtype=torch.float64).reshape(t.shape)
                                   .remainder(97.0)).sum())
    return cs


def run_reference(name):
    V = ref_loader.load()[0]
    inp = build_inputs(name)
    c = inp["case"]
    dense = inp["dense"].clone().requires_grad_(True)
    with contextlib.redirect_stdout(io.StringIO()):
        m = V.Sins(SR, P, c["H"], c["Ma"], c["Mn"], n_unit=8)
    m.unit2ctrl = ref_loader.fixed_ctrl_module(syn.split_views(dense, split_map(name)), torch.zeros(c["B"], c["nF"], 256))
    torch.manual_seed(G.seeds(name)["noise"])
    signal, _, (harmonic, noise) = m(None, inp["f0"], None, infer=False)
    objective(signal, harmonic, noise, inp).backward()
    return inp, {"grad": dense.grad, "signal": signal.detach()}


def main():
    if not ref_loader.available():
        raise SystemExit("live reference not found; set DDSP_REFERENCE_ROOT to a DDSP-SVC checkout")
    for name in sys.argv[1:] or CASES:
        inp, out = run_reference(name)
        payload = {k: v.numpy().astype(np.float32) for k, v in out.items()}
        payload.update({k: np.float64(v) for k, v in input_checksums(inp).items()})
        payload["torch_version"] = np.array(torch.__version__)
        np.savez_compressed(path(name), **payload)
        print("%-36s %s" % (name, {k: tuple(v.shape) for k, v in payload.items() if getattr(v, "ndim", 0) > 0}))


if __name__ == "__main__":
    main()
