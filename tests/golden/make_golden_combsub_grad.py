"""Generate tests/golden/combsub_grad_*.npz: the LIVE reference's own autograd gradient of the old CombSub (training
phase, infer=False) with respect to its three raw controls, on CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_combsub_grad.py [case names; default: all]

As make_golden_sins_grad.py: the reference's Unit2Control is replaced by a module returning views of one leaf
``dense`` tensor that requires grad (the split_to_dict layout), the noise is pinned by torch.manual_seed(seed) right
before forward(), then ``(signal * cot + harmonic * cot_h + noise * cot_n).sum().backward()`` with seeded cotangents
(cot_h / cot_n only where the case says so).  Each .npz stores dense.grad [B, nF, Ma + Mh + Mn], the signal, and
float64 checksums of every input.

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
from tests.golden import make_golden_sins_grad as GS  # noqa: E402

SR, P = G.SR, G.P

CASES = OrderedDict([
    # the reference's CombSub shape; unvoiced frames and a 65 -> 1100 Hz sweep row (harmonics cross Nyquist)
    ("combsub_grad_b2_f24", dict(B=2, nF=24, Ma=256, Mh=512, Mn=256, unvoiced=0.1, sweep_row=1)),
    ("combsub_grad_b1_f1", dict(B=1, nF=1, Ma=256, Mh=512, Mn=256)),
    ("combsub_grad_b1_f2", dict(B=1, nF=2, Ma=256, Mh=512, Mn=256)),
    # Ma != Mn: the forward's separate all-pass / noise FIR launches
    ("combsub_grad_b1_f5_ma65_mh129_mn33", dict(B=1, nF=5, Ma=65, Mh=129, Mn=33)),
    ("combsub_grad_b1_f4_ma2_mh3_mn2", dict(B=1, nF=4, Ma=2, Mh=3, Mn=2)),
    # exactly 1024 harmonic taps
    ("combsub_grad_b1_f3_mh513", dict(B=1, nF=3, Ma=256, Mh=513, Mn=256)),
    # cotangents on harmonic and noise as well as on signal
    ("combsub_grad_b2_f6_parts", dict(B=2, nF=6, Ma=256, Mh=512, Mn=256, parts=True)),
    # a longer utterance: the comb's phase difference grows with length
    ("combsub_grad_b1_f70", dict(B=1, nF=70, Ma=256, Mh=512, Mn=256)),
])


def path(name):
    return os.path.join(G.HERE, name + ".npz")


def split_map(name):
    c = CASES[name]
    return syn.combsub_split_map(c["Ma"], c["Mh"], c["Mn"])


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


objective = GS.objective
input_checksums = GS.input_checksums


def run_reference(name):
    V = ref_loader.load()[0]
    inp = build_inputs(name)
    c = inp["case"]
    dense = inp["dense"].clone().requires_grad_(True)
    with contextlib.redirect_stdout(io.StringIO()):
        m = V.CombSub(SR, P, c["Ma"], c["Mh"], c["Mn"], n_unit=8)
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
