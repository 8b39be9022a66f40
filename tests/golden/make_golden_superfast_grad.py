"""Generate tests/golden/superfast_grad_*.npz: the LIVE reference's own autograd gradient of CombSubSuperFast with
respect to its four raw controls, on CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_superfast_grad.py [case names; default: all]

The reference's Unit2Control is replaced by a module returning views of one leaf ``dense`` tensor that requires
grad (the split_to_dict layout, ddsp/unit2control.py:12-23); noise is pinned by torch.manual_seed(seed) right before
forward(), as make_golden.py does; then ``(signal * cot).sum().backward()`` with a seeded cotangent ``cot``.  Each
.npz stores dense.grad [B, nF, 4*1025], the signal, and float64 checksums of every input.

The case list lives here (not in cases.py, whose superfast cases other tests loop over); the tests import
``CASES`` / ``build_inputs`` from this module and only read the stored files.
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

SR, P, WIN = G.SR, G.P, 2048

CASES = OrderedDict([
    # unvoiced frames (f0 = 0: the s + 1e-5 path) and one 65 -> 1100 Hz sweep row
    ("superfast_grad_b2_f24", dict(B=2, nF=24, unvoiced=0.1, sweep_row=1)),
    ("superfast_grad_b1_f5", dict(B=1, nF=5)),
    ("superfast_grad_b1_f2_constpad", dict(B=1, nF=2)),       # T <= 1024: constant padding
    ("superfast_grad_b1_f1", dict(B=1, nF=1)),                # both STFT frames use control row 0
    ("superfast_grad_b1_f48", dict(B=1, nF=48)),              # several kernel chunks (2 of 29 hops, 10 of 5)
])


def path(name):
    return os.path.join(G.HERE, name + ".npz")


def split_map():
    return syn.superfast_split_map(WIN)


def build_inputs(name):
    """f0 [B, nF, 1], dense raw controls [B, nF, 4*1025] + split views, N(0,1) noise [B, T], cotangent [B, T]."""
    case = CASES[name]
    sd = G.seeds(name)
    B, nF = case["B"], case["nF"]
    f0 = syn.make_f0(B, nF, SR, P, seed=sd["f0"], unvoiced_fraction=case.get("unvoiced", 0.0),
                     sweep_row=case.get("sweep_row"))
    dense, views = syn.make_ctrl(B, nF, split_map(), seed=sd["ctrl"])
    noise = syn.normal_noise((B, nF * P), sd["noise"])
    cot = torch.randn(B, nF * P, generator=torch.Generator().manual_seed(sd["noise"] + 1000))
    return {"case": case, "f0": f0, "dense": dense, "ctrls": views, "noise": noise, "cot": cot}


def input_checksums(inp):
    """cases.input_checksums (f0, dense, noise) plus the same checksum of the cotangent"""
    cs = G.input_checksums(inp)
    t = inp["cot"].double()
    cs["cs_cot"] = float((t * torch.arange(1, t.numel() + 1, dtype=torch.float64).reshape(t.shape).remainder(97.0)).sum())
    return cs


def run_reference(name):
    V = ref_loader.load()[0]
    inp = build_inputs(name)
    B, nF = inp["case"]["B"], inp["case"]["nF"]
    dense = inp["dense"].clone().requires_grad_(True)
    with contextlib.redirect_stdout(io.StringIO()):
        m = V.CombSubSuperFast(SR, P, WIN, n_unit=8)
    m.eval()
    m.unit2ctrl = ref_loader.fixed_ctrl_module(syn.split_views(dense, split_map()), torch.zeros(B, nF, 256))
    torch.manual_seed(G.seeds(name)["noise"])
    signal, _, _ = m(None, inp["f0"], None)
    (signal * inp["cot"]).sum().backward()
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
        print("%-32s %s" % (name, {k: tuple(v.shape) for k, v in payload.items() if getattr(v, "ndim", 0) > 0}))


if __name__ == "__main__":
    main()
