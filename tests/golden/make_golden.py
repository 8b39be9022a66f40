"""Generate tests/golden/*.npz by running the LIVE reference (yxlllc/DDSP-SVC) on CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden.py

The reference's Unit2Control is replaced by a module returning the fixed raw controls
(the DSP/NN seam, ddsp/vocoder.py:578/664/832); noise is pinned by calling
torch.manual_seed(seed) right before forward(), which makes the reference's internal
rand_like / randn_like equal to the tensor the tests feed to the CUDA path explicitly
(SURVEY.md appendix B).
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests.golden import cases as G  # noqa: E402


def run_reference(name):
    V, _, SineGen = ref_loader.load()
    inp = G.build_inputs(name)
    case = inp["case"]
    sd = G.seeds(name)
    B, nF = case["B"], case["nF"]
    hidden = torch.zeros(B, nF, 256)
    out = {}
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        if case["kind"] == "sinegen":
            gen = SineGen(G.SR, harmonic_num=case["harmonic_num"])
            torch.manual_seed(sd["noise"])
            out["out"] = gen(inp["f0"], case["upp"])
        elif case["kind"] == "source_module":
            import nsf_hifigan.models as ref_nsf
            torch.manual_seed(sd["ctrl"])                       # seeds the Linear(9 -> 1) initialisation
            m = ref_nsf.SourceModuleHnNSF(G.SR, harmonic_num=case["harmonic_num"])
            torch.manual_seed(sd["noise"])
            out["out"] = m(inp["f0"], case["upp"])
            out["weight"] = m.l_linear.weight.detach().clone()
            out["bias"] = m.l_linear.bias.detach().clone()
        else:
            if case["kind"] == "sins":
                m = V.Sins(G.SR, G.P, case["H"], case["Ma"], case["Mn"], n_unit=8)
            elif case["kind"] == "combsub":
                m = V.CombSub(G.SR, G.P, case["Ma"], case["Mh"], case["Mn"], n_unit=8)
            elif case["kind"] == "combsubfast":
                m = V.CombSubFast(G.SR, G.P, n_unit=8)
            else:
                m = V.CombSubSuperFast(G.SR, G.P, case["win"], n_unit=8)
            m.eval()
            seen = {}

            class Ctrl(torch.nn.Module):
                def forward(self, units, f0, phase, volume, **kw):
                    seen["phase_frames"] = phase.clone()
                    return inp["ctrls"], hidden

            m.unit2ctrl = Ctrl()
            torch.manual_seed(sd["noise"])
            kw = {}
            if "initial_phase" in inp:
                kw["initial_phase"] = inp["initial_phase"]
            signal, _, (harm, noise) = m(None, inp["f0"], None, **kw)
            out.update(signal=signal, harmonic=harm, noise=noise, phase_frames=seen["phase_frames"])
    return inp, out


def main():
    if not ref_loader.available():
        raise SystemExit("live reference not found; goldens can only be regenerated in the build container")
    for name, case in G.CASES.items():
        inp, out = run_reference(name)
        payload = {k: out[k].numpy().astype(np.float32) for k in tuple(case["store"]) + tuple(case.get("extra", ()))}
        payload.update({k: np.float64(v) for k, v in G.input_checksums(inp).items()})
        payload["torch_version"] = np.array(torch.__version__)
        np.savez_compressed(G.path(name), **payload)
        print("%-36s %s" % (name, {k: tuple(v.shape) for k, v in payload.items() if getattr(v, "ndim", 0) > 0}))


if __name__ == "__main__":
    main()
