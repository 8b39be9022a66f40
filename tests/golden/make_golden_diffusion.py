"""Generate tests/golden/diffusion_*.npz: the LIVE reference's GaussianDiffusion (diffusion/diffusion.py) with its five
samplers around the WaveNet denoiser (diffusion/wavenet.py) and around NaiveV2Diff (diffusion/naive_v2_diff.py, as
Unit2WavFast builds it), on the CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_diffusion.py [case names; default: all]

diffusion/diffusion.py imports librosa.sequence, which it never uses; where librosa is not installed the generator puts
an empty stand-in module in its place before importing (here only: the other drop-in tests see the modules as they are).

Weights are not stored: ``build_oracle`` rebuilds them from a seed (tests/reflow_oracle.seeded_weights: every parameter
non-zero -- the reference zero-initialises the output projection, which would make the noise prediction a constant).
Each sampler file holds the inputs, the start's draw ``noise`` [B, 1, M, T] (torch.randn, or randn_like of the
transposed view for the shallow start) and DDPM's per-step draws ``step_noise`` under ``torch.manual_seed(seed)``, in
the reference's order, the diffusion-step values the network was called with (``fed``, first utterance) and the
reference's fp32 output ``out32``.  The standalone-network files hold ``out32`` and ``out64`` (the module in float64).

The reference's PNDM takes ``max(t - interval, 0)`` of a [B] tensor, which raises for B > 1: its case runs at B = 1.
"""
import os
import sys
import types
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import diffusion_oracle, reflow_oracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# a small WaveNet, the configs' WaveNet(128, 20, 512, 256), and a small NaiveV2Diff (mel 128, condition 128)
MODELS = OrderedDict([("w64", dict(kind="wavenet", n_layers=3, n_chans=64, n_hidden=256, seed=31)),
                      ("w512", dict(kind="wavenet", n_layers=20, n_chans=512, n_hidden=256, seed=32)),
                      ("naive", dict(kind="naive", dim=128, num_layers=2, cond=128, seed=33))])

CASES = OrderedDict([
    ("diffusion_w64_b2_t24_dpm10", dict(model="w64", B=2, T=24, method="dpm-solver", speedup=10, k_step=100)),
    ("diffusion_w64_b2_t17_unipc10", dict(model="w64", B=2, T=17, method="unipc", speedup=10, k_step=100)),
    ("diffusion_w64_b1_t20_pndm10", dict(model="w64", B=1, T=20, method="pndm", speedup=10, k_step=100)),
    ("diffusion_w64_b2_t9_ddim10", dict(model="w64", B=2, T=9, method="ddim", speedup=10, k_step=100)),
    ("diffusion_w64_b1_t12_ddpm", dict(model="w64", B=1, T=12, method=None, speedup=10, k_step=100)),
    # fewer than 10 steps: DPM-Solver's first-order final step; UniPC with 2 steps
    ("diffusion_w64_b2_t15_dpm25", dict(model="w64", B=2, T=15, method="dpm-solver", speedup=25, k_step=100)),
    ("diffusion_w64_b1_t11_unipc34", dict(model="w64", B=1, T=11, method="unipc", speedup=34, k_step=100)),
    # the full-noise start from t = k_step (1000): no gt_spec
    ("diffusion_w64_b2_t10_dpm100_nogt", dict(model="w64", B=2, T=10, method="dpm-solver", speedup=100, k_step=None)),
    ("diffusion_w512_b1_t16_dpm10", dict(model="w512", B=1, T=16, method="dpm-solver", speedup=10, k_step=100)),
    ("diffusion_w512_b1_t13_unipc10", dict(model="w512", B=1, T=13, method="unipc", speedup=10, k_step=100)),
    ("diffusion_naive_b2_t14_dpm10", dict(model="naive", B=2, T=14, method="dpm-solver", speedup=10, k_step=100)),
    ("diffusion_naive_b1_t10_pndm10", dict(model="naive", B=1, T=10, method="pndm", speedup=10, k_step=100)),
    # the standalone network at float steps, one per utterance
    ("diffusion_net_w64_b2_t1", dict(model="w64", B=2, T=1, net=True, step=[37.5, 912.25])),
    ("diffusion_net_w512_b2_t13", dict(model="w512", B=2, T=13, net=True, step=[99.0, 0.5])),
])


def path(name):
    return os.path.join(HERE, name + ".npz")


def _seed(name):
    return 3000 + list(CASES).index(name)


def mel_channels(model):
    return 128


def cond_channels(model):
    m = MODELS[model]
    return m["n_hidden"] if m["kind"] == "wavenet" else m["cond"]


def build_oracle(model):
    """the oracle network with the model's seeded weights (fp32, CPU): diffusion_oracle.WaveNet or
    reflow_oracle.VelocityNet"""
    m = MODELS[model]
    if m["kind"] == "wavenet":
        net = diffusion_oracle.WaveNet(128, m["n_layers"], m["n_chans"], m["n_hidden"])
    else:
        net = reflow_oracle.VelocityNet(128, m["dim"], m["cond"], m["num_layers"])
    return reflow_oracle.seeded_weights(net, m["seed"])


def package_kwargs(model):
    """constructor arguments of the package's (and the reference's) denoiser: (class name, kwargs)"""
    m = MODELS[model]
    if m["kind"] == "wavenet":
        return "WaveNet", dict(in_dims=128, n_layers=m["n_layers"], n_chans=m["n_chans"], n_hidden=m["n_hidden"])
    return "NaiveV2Diff", dict(mel_channels=128, dim=m["dim"], num_layers=m["num_layers"], condition_dim=m["cond"],
                               use_mlp=False)


def build_inputs(name):
    """condition [B, T, M_cond] and gt_spec [B, T, M] (log-mel-like: a ramp over the bins plus noise); network cases:
    spec [B, 1, M, T], step [B], cond [B, M_cond, T]"""
    c = CASES[name]
    g = torch.Generator().manual_seed(_seed(name))
    B, T, Mc = c["B"], c["T"], cond_channels(c["model"])
    cramp = torch.linspace(-8.0, 0.5, Mc)[None, None, :]
    condition = cramp + 1.5 * torch.randn(B, T, Mc, generator=g)
    if c.get("net"):
        return dict(spec=torch.randn(B, 1, 128, T, generator=g), step=torch.tensor(c["step"]),
                    cond=condition.transpose(1, 2).contiguous())
    ramp = torch.linspace(-8.0, 0.5, 128)[None, None, :]
    return dict(condition=condition, gt_spec=ramp + 1.5 * torch.randn(B, T, 128, generator=g))


def _reference():
    ref_loader.load()                                  # the checkout on sys.path with its stub modules
    try:
        import librosa.sequence  # noqa: F401
    except ImportError:                                # diffusion.py imports it and never uses it
        sys.modules.setdefault("librosa", types.ModuleType("librosa"))
        sys.modules.setdefault("librosa.sequence", types.ModuleType("librosa.sequence"))
    import diffusion.diffusion as dd
    import diffusion.naive_v2_diff as nv
    import diffusion.wavenet as wn
    return dd, wn, nv


def build_reference(model):
    _, wn, nv = _reference()
    cls, kw = package_kwargs(model)
    net = wn.WaveNet(**kw) if cls == "WaveNet" else nv.NaiveV2Diff(**kw)
    net.load_state_dict(build_oracle(model).state_dict(), strict=True)
    return net.eval()


def generate(name):
    c = CASES[name]
    dd, _, _ = _reference()
    net = build_reference(c["model"])
    inp = build_inputs(name)
    out = {k: v.numpy() for k, v in inp.items()}
    with torch.no_grad():
        if c.get("net"):
            out["out32"] = net(inp["spec"], inp["step"], inp["cond"]).numpy()
            out["out64"] = net.double()(inp["spec"].double(), inp["step"].double(), inp["cond"].double()).numpy()
            np.savez_compressed(path(name), **out)
            return
        gd = dd.GaussianDiffusion(net, out_dims=128)
        fed, orig = [], net.forward

        def spy(spec, t, cond):
            fed.append(float(torch.as_tensor(t).reshape(-1)[0]))
            return orig(spec, t, cond)
        net.forward = spy
        kw = dict(infer=True, infer_speedup=c["speedup"], method=c["method"], k_step=c["k_step"], use_tqdm=False)
        gt = inp["gt_spec"] if c["k_step"] is not None else None
        torch.manual_seed(_seed(name))
        out["out32"] = gd(inp["condition"], gt_spec=gt, **kw).numpy()
        out["fed"] = np.array(fed)
        # the same draws again, in the reference's order: the start, then DDPM's one randn per step
        B, T = c["B"], c["T"]
        torch.manual_seed(_seed(name))
        if gt is None:
            t, noise = gd.k_step, torch.randn((B, 1, 128, T))
        else:
            t, noise = c["k_step"], torch.randn_like(gd.norm_spec(gt).transpose(1, 2)[:, None, :, :])
        out["noise"] = np.ascontiguousarray(noise.numpy())
        if c["method"] is None or c["speedup"] == 1:
            out["step_noise"] = torch.stack([torch.randn((B, 1, 128, T)) for _ in range(t)]).numpy()
    if gt is None:
        out.pop("gt_spec")
    np.savez_compressed(path(name), **out)


def write_state_dict_keys():
    """diffusion_state_dicts.json: [key, shape] of the reference's denoisers (each model), of GaussianDiffusion around
    them and of the configs' WaveNet(128, 20, 512, 256) / NaiveV2Diff(128, 512, 6 layers) as Unit2Wav / Unit2WavFast
    hold them"""
    import json
    dd, wn, nv = _reference()
    shapes = lambda m: [[k, list(v.shape)] for k, v in m.state_dict().items()]
    sd = {m: shapes(build_reference(m)) for m in MODELS}
    sd["GaussianDiffusion_w64"] = shapes(dd.GaussianDiffusion(build_reference("w64"), out_dims=128))
    sd["Unit2Wav.diff_model"] = shapes(dd.GaussianDiffusion(wn.WaveNet(128, 20, 512, 256), out_dims=128))
    sd["Unit2WavFast.diff_model"] = shapes(dd.GaussianDiffusion(
        nv.NaiveV2Diff(mel_channels=128, dim=512, num_layers=6, condition_dim=128, use_mlp=False), out_dims=128))
    with open(os.path.join(HERE, "diffusion_state_dicts.json"), "w") as f:
        json.dump(sd, f)


def buffer_values():
    """the reference's registered buffers of GaussianDiffusion (defaults), by name -> float64 numpy"""
    dd, _, _ = _reference()
    gd = dd.GaussianDiffusion(build_reference("w64"), out_dims=128)
    return {k: v.double().numpy() for k, v in gd.named_buffers()}


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    write_state_dict_keys()
    np.savez_compressed(os.path.join(HERE, "diffusion_buffers.npz"), **buffer_values())
    for n in names:
        generate(n)
        d = np.load(path(n))
        print("wrote", path(n), "out32 rms %.3f" % float(np.sqrt((d["out32"] ** 2).mean())),
              "evaluations", len(d["fed"]) if "fed" in d else "-")
