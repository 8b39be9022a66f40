"""Generate tests/golden/units_*.npz: the LIVE reference's units encoder on the CPU in float64.

Cases: ``HubertSoft.units`` (encoder/hubert/model.py) at 400 samples (one frame), 0.5 s and 2 s with B = 1 and 2, a
silent clip (GroupNorm with zero variance) and a case whose q / k projections are scaled so attention is peaked (the
median of the largest attention probability of the first layer above 0.5); and the reference's
``Units_Encoder('hubertsoft', ...).encode`` (ddsp/vocoder.py) at 16 kHz / hop 320, at 44.1 kHz / hop 512 and with 1000
samples at 44.1 kHz (363 resampled samples: the reference then pads the unresampled audio to 1037).

The weights (94 M parameters) are never stored: they come from tests/units_oracle.seeded_state_dict and each file
holds the float64 sum of the ones it was made with, checked by ``load``.  Inputs and outputs are stored in fp32 (the
outputs are float64 results rounded once).  One thread: regenerating gives byte-identical files.

Run from the repository root with DDSP_REFERENCE_ROOT pointing at a reference checkout:
    python tests/golden/make_golden_units.py [case ...]
"""
import os
import sys
import tempfile
import types
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import units_oracle as U  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
WEIGHTS = OrderedDict([("soft", dict(seed=41, peaked=False)), ("peaked", dict(seed=42, peaked=True))])
CASES = OrderedDict()
for _B in (1, 2):
    for _n in (400, 8000, 32000):
        CASES["units_soft_b%d_n%d" % (_B, _n)] = dict(kind="units", weights="soft", B=_B, n=_n)
CASES["units_soft_silent"] = dict(kind="units", weights="soft", B=1, n=8000, silent=True)
CASES["units_peaked_b1_n8000"] = dict(kind="units", weights="peaked", B=1, n=8000)
CASES["units_encode_16000"] = dict(kind="encode", weights="soft", B=1, n=16000 + 37, sr=16000, hop=320)
CASES["units_encode_44100"] = dict(kind="encode", weights="soft", B=1, n=44100 + 211, sr=44100, hop=512)
CASES["units_encode_44100_n1000"] = dict(kind="encode", weights="soft", B=1, n=1000, sr=44100, hop=512)


def path(name):
    return os.path.join(HERE, name + ".npz")


def weights_sum(sd):
    return float(sum(v.double().sum() for v in sd.values() if v.is_floating_point()))


def weights(name, expected_sum=None):
    """the seeded HubertSoft state dict of WEIGHTS[name] (fp32, CPU); checks ``expected_sum`` when given"""
    sd = U.seeded_state_dict(**WEIGHTS[name])
    if expected_sum is not None:
        got = weights_sum(sd)
        assert abs(got - expected_sum) <= 1e-9 * max(1.0, abs(expected_sum)), (got, expected_sum)
    return sd


def load(name):
    """the golden of case ``name`` as a dict of numpy arrays / scalars, and its state dict with the weights checked"""
    with np.load(path(name)) as z:
        d = {k: z[k] for k in z.files}
    return d, weights(str(d["weights"]), float(d["weights_sum"]))


def audio(name):
    spec = CASES[name]
    if spec.get("silent"):
        return torch.zeros(spec["B"], spec["n"])
    g = torch.Generator().manual_seed(6000 + list(CASES).index(name))
    return torch.randn(spec["B"], spec["n"], generator=g) * 0.3


def reference():
    V = ref_loader.load()[0]
    if "sklearn.cluster" not in sys.modules:          # encoder.hubert.model imports KMeans for HubertDiscrete only
        try:
            import sklearn.cluster  # noqa: F401
        except ImportError:
            sys.modules.setdefault("sklearn", types.ModuleType("sklearn"))
            sys.modules["sklearn.cluster"] = types.SimpleNamespace(KMeans=object)
    from encoder.hubert import model as M
    return V, M


def _peaked_enough(sd, x):
    """median over queries and heads of the largest attention probability of layer 0, in float64 (the oracle)"""
    import torch.nn.functional as F
    h = U.features(sd, F.pad(x.double(), (40, 40)))
    h = F.layer_norm(h + U.positional(sd, h), (768,), sd["norm.weight"].double(), sd["norm.bias"].double(), 1e-5)
    qkv = F.linear(h, sd["encoder.layers.0.self_attn.in_proj_weight"].double(),
                   sd["encoder.layers.0.self_attn.in_proj_bias"].double())
    q, k, _ = (t.reshape(h.shape[0], -1, 12, 64).transpose(1, 2) for t in qkv.split(768, -1))
    return torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1).max(-1).values.median().item()


def make(name, V, M):
    spec = CASES[name]
    sd = weights(spec["weights"])
    x = audio(name)
    out = dict(weights=spec["weights"], weights_sum=weights_sum(sd), audio=x.numpy())
    with torch.inference_mode():
        if spec["kind"] == "units":
            ref = M.HubertSoft()
            ref.load_state_dict(sd)
            units = ref.double().eval().units(x.double()[:, None])
        else:
            tmp = tempfile.mkdtemp()
            ckpt = os.path.join(tmp, "hubert-soft.pt")
            torch.save({"module." + k: v for k, v in sd.items()}, ckpt)   # the released file's DataParallel prefix
            enc = V.Units_Encoder("hubertsoft", ckpt, device="cpu")
            os.remove(ckpt)
            os.rmdir(tmp)
            enc.model.hubert.double()
            if spec["sr"] != 16000:
                enc.resample_kernel[str(spec["sr"])] = V.Resample(spec["sr"], 16000, lowpass_filter_width=128).to(
                    torch.float64)
            units = enc.encode(x.double(), spec["sr"], spec["hop"])
            out.update(sr=spec["sr"], hop=spec["hop"])
    if spec["weights"] == "peaked":
        p = _peaked_enough(sd, x)
        assert p > 0.5, p
    out["units"] = units.float().numpy()
    np.savez(path(name), **out)
    print("wrote", path(name), os.path.getsize(path(name)), "bytes", tuple(units.shape))


def main(names):
    torch.set_num_threads(1)                       # a fixed summation order: byte-identical regeneration
    V, M = reference()
    for name in names or CASES:
        make(name, V, M)


if __name__ == "__main__":
    main(sys.argv[1:])
