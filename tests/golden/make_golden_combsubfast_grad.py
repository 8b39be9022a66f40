"""Generate tests/golden/csfast_grad_*.npz: the LIVE reference's own autograd gradient of CombSubFast (training phase,
infer=False, as diffusion/solver_new.py runs it) with respect to its three raw controls, on CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_combsubfast_grad.py [case names; default: all]

The reference's Unit2Control is replaced by a module returning views of one leaf ``dense`` tensor that requires grad
(the split_to_dict layout, ddsp/unit2control.py:12-23); the noise is pinned by torch.manual_seed(seed) right before
forward(), so that synthetic.uniform_noise reproduces rand_like; then ``(signal * cot).sum().backward()`` with a
seeded cotangent ``cot``.  Each .npz stores dense.grad [B, nF, 3*513], the signal, float64 checksums of every
input, and the fingerprint of the FFT code path that computed them (``fft_fingerprint``).

The case list lives here; the tests import ``CASES`` / ``build_inputs`` from this module and only read the stored files.
"""
import contextlib
import hashlib
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
NB = P + 1

CASES = OrderedDict([
    # unvoiced frames (f0 = 0) and one 65 -> 1100 Hz sweep row
    ("csfast_grad_b2_f24", dict(B=2, nF=24, unvoiced=0.1, sweep_row=1)),
    ("csfast_grad_b1_f1", dict(B=1, nF=1)),                     # frames 0 and 1 both use control row 0
    ("csfast_grad_b1_f2", dict(B=1, nF=2)),                     # frame nF = 2 alone in its pair
    ("csfast_grad_b1_f3_unvoiced", dict(B=1, nF=3, unvoiced=0.4)),
    # initial_phase is added to the fp32 cumsum in the training phase (a second rounding of the phase)
    ("csfast_grad_b1_f9_initphase", dict(B=1, nF=9, initial_phase=True)),
    ("csfast_grad_b1_f70", dict(B=1, nF=70)),                   # two full 32-row chunks and a ragged one
])


def path(name):
    return os.path.join(G.HERE, name + ".npz")


def split_map():
    return syn.combsubfast_split_map(P)


def build_inputs(name):
    """f0 [B, nF, 1], dense raw controls [B, nF, 3*513] + split views, U(-1, 1) noise [B, T], cotangent [B, T],
    initial_phase [B, 1, 1] or None."""
    case = CASES[name]
    sd = G.seeds(name)
    B, nF = case["B"], case["nF"]
    f0 = syn.make_f0(B, nF, SR, P, seed=sd["f0"], unvoiced_fraction=case.get("unvoiced", 0.0),
                     sweep_row=case.get("sweep_row"))
    dense, views = syn.make_ctrl(B, nF, split_map(), seed=sd["ctrl"])
    noise = syn.uniform_noise(B, nF * P, sd["noise"])
    cot = torch.randn(B, nF * P, generator=torch.Generator().manual_seed(sd["noise"] + 1000))
    initial_phase = None
    if case.get("initial_phase"):
        g = torch.Generator().manual_seed(sd["noise"] + 1)
        initial_phase = torch.rand(B, 1, 1, generator=g) * 6.0 - 3.0
    return {"case": case, "f0": f0, "dense": dense, "ctrls": views, "noise": noise, "cot": cot,
            "initial_phase": initial_phase}


def fft_fingerprint():
    """Hash of a seeded 1024-point rfft / irfft on this machine.  torch's CPU FFT (MKL) picks its code path from the
    instruction set, and paths differ in the last bits, so the goldens are the reference's bits only where this
    matches the value stored with them."""
    x = torch.randn(3, 2 * P, generator=torch.Generator().manual_seed(0))
    s = torch.fft.rfft(x, 2 * P)
    y = torch.fft.irfft(s * (1 + 0.5j), 2 * P)
    return hashlib.sha256(s.numpy().tobytes() + y.numpy().tobytes()).hexdigest()


def input_checksums(inp):
    """cases.input_checksums (f0, dense, noise, initial_phase) plus the same checksum of the cotangent"""
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
        m = V.CombSubFast(SR, P, n_unit=8)
    m.unit2ctrl = ref_loader.fixed_ctrl_module(syn.split_views(dense, split_map()), torch.zeros(B, nF, 256))
    torch.manual_seed(G.seeds(name)["noise"])
    signal, _, _ = m(None, inp["f0"], None, initial_phase=inp["initial_phase"], infer=False)
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
        payload["fft_fingerprint"] = np.array(fft_fingerprint())
        np.savez_compressed(path(name), **payload)
        print("%-32s %s" % (name, {k: tuple(v.shape) for k, v in payload.items() if getattr(v, "ndim", 0) > 0}))


if __name__ == "__main__":
    main()
