"""Generate tests/golden/reflow_*.npz: the LIVE reference's velocity network NaiveV2Diff (reflow/naive_v2_diff.py,
use_mlp=False as Unit2Wav builds it) and its RectifiedFlow sampler (reflow/reflow.py) on the CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_reflow.py [case names; default: all]

Weights are not stored: ``build_reference`` / ``MODELS`` rebuild them from a seed (tests/reflow_oracle.seeded_weights:
every parameter non-zero -- the reference zero-initialises the output projection, which would make the velocity a
constant -- scaled so each layer's residual update is of the order of its input).  Each file holds the inputs, the
noise the sampler drew under ``torch.manual_seed(seed)`` (one torch.randn of [B, 1, M, T], the reference's draw) and
the reference's fp32 output ``out32``; the velocity cases also hold ``out64``, the reference module in float64.

The reference's ``gt_spec=None`` start creates t with ``torch.full((b,), 0)``, an int64 tensor, so its first
``t += dt`` raises RuntimeError; the generator checks that it still does and stores, for those cases, the reference's
own sample_euler / sample_rk4 steps driven from an fp32 t = 0 (what the branch means).  ``infer_step=0`` divides by zero
in the reference (ZeroDivisionError); the case stores only that fact.
"""
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import reflow_oracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# width 128 with 2 layers, and the reflow.yaml stack (n_chans 512, n_layers 6); 128 mel bins, condition 128 as in Unit2Wav
MODELS = OrderedDict([("w128", dict(dim=128, num_layers=2, mel=128, cond=128, seed=11)),
                      ("w512", dict(dim=512, num_layers=6, mel=128, cond=128, seed=12))])

CASES = OrderedDict([
    ("reflow_w128_b1_t37_euler5_t07", dict(model="w128", B=1, T=37, method="euler", steps=5, gt=True, t_start=0.7)),
    ("reflow_w128_b2_t70_rk4_3_t0", dict(model="w128", B=2, T=70, method="rk4", steps=3, gt=True, t_start=0.0)),
    ("reflow_w128_b2_t8_euler4_nogt", dict(model="w128", B=2, T=8, method="euler", steps=4, gt=False, t_start=0.0)),
    ("reflow_w128_b1_t20_rk4_3_nogt", dict(model="w128", B=1, T=20, method="rk4", steps=3, gt=False, t_start=0.0)),
    ("reflow_w128_b2_t12_rk4_4_t07", dict(model="w128", B=2, T=12, method="rk4", steps=4, gt=True, t_start=0.7)),
    ("reflow_w128_b1_t9_euler0_t07", dict(model="w128", B=1, T=9, method="euler", steps=0, gt=True, t_start=0.7)),
    ("reflow_w512_b1_t24_euler3_t07", dict(model="w512", B=1, T=24, method="euler", steps=3, gt=True, t_start=0.7)),
    ("reflow_w512_b2_t16_rk4_3_nogt", dict(model="w512", B=2, T=16, method="rk4", steps=3, gt=False, t_start=0.0)),
    # the standalone velocity network: 4-dim and 3-dim spec, one diffusion step per utterance
    ("reflow_vel_w128_b2_t33", dict(model="w128", B=2, T=33, velocity=True, four=True, step=[123.25, 870.5])),
    ("reflow_vel_w512_b1_t19", dict(model="w512", B=1, T=19, velocity=True, four=False, step=[431.0])),
])


def path(name):
    return os.path.join(HERE, name + ".npz")


def _seed(name):
    return 2000 + list(CASES).index(name)


def model_kwargs(model):
    m = MODELS[model]
    return dict(mel_channels=m["mel"], dim=m["dim"], condition_dim=m["cond"], num_layers=m["num_layers"])


def build_oracle(model):
    """tests/reflow_oracle.VelocityNet with the model's seeded weights (fp32, CPU)"""
    m = MODELS[model]
    net = reflow_oracle.VelocityNet(m["mel"], m["dim"], m["cond"], m["num_layers"])
    return reflow_oracle.seeded_weights(net, m["seed"])


def build_inputs(name):
    """condition [B, T, M_cond] (a smooth log-mel-like signal), gt_spec [B, T, M] or None; velocity cases: spec
    [B, 1, M, T] or [B, M, T], step [B], cond [B, M_cond, T]"""
    c, m = CASES[name], MODELS[CASES[name]["model"]]
    g = torch.Generator().manual_seed(_seed(name))
    B, T = c["B"], c["T"]
    ramp = torch.linspace(-8.0, 0.5, m["cond"])[None, None, :]
    condition = ramp + 1.5 * torch.randn(B, T, m["cond"], generator=g)
    if c.get("velocity"):
        spec = torch.randn(B, m["mel"], T, generator=g)
        return dict(spec=spec[:, None] if c["four"] else spec, step=torch.tensor(c["step"]),
                    cond=condition.transpose(1, 2).contiguous())
    gt = ramp[..., :m["mel"]] + 1.5 * torch.randn(B, T, m["mel"], generator=g) if c["gt"] else None
    return dict(condition=condition, gt_spec=gt)


def _reference():
    ref_loader.load()                                  # puts the checkout on sys.path with its stub modules
    import reflow.naive_v2_diff as nv
    import reflow.reflow as rf
    return nv, rf


def build_reference(model):
    nv, _ = _reference()
    net = nv.NaiveV2Diff(use_mlp=False, **model_kwargs(model))
    net.load_state_dict(build_oracle(model).state_dict(), strict=True)
    return net


def generate(name):
    c = CASES[name]
    nv, rf = _reference()
    net = build_reference(c["model"]).eval()
    inp = build_inputs(name)
    out = {k: v.numpy() for k, v in inp.items() if v is not None}
    with torch.no_grad():
        if c.get("velocity"):
            out["out32"] = net(inp["spec"], inp["step"], inp["cond"]).numpy()
            out["out64"] = net.double()(inp["spec"].double(), inp["step"].double(), inp["cond"].double()).numpy()
            np.savez_compressed(path(name), **out)
            return
        flow = rf.RectifiedFlow(net, out_dims=MODELS[c["model"]]["mel"])
        B, T = c["B"], c["T"]
        shape = (B, 1, MODELS[c["model"]]["mel"], T)
        torch.manual_seed(_seed(name))
        out["noise"] = torch.randn(shape).numpy()
        kw = dict(infer=True, infer_step=c["steps"], method=c["method"], t_start=c["t_start"], use_tqdm=False)
        torch.manual_seed(_seed(name))
        if c["steps"] == 0:
            try:
                flow(inp["condition"], gt_spec=inp["gt_spec"], **kw)
            except ZeroDivisionError:
                out["raises"] = np.array("ZeroDivisionError")
            else:
                raise AssertionError("the reference no longer divides by zero at infer_step=0")
        elif inp["gt_spec"] is None:
            try:
                flow(inp["condition"], gt_spec=None, **kw)
            except RuntimeError:
                pass
            else:
                raise AssertionError("the reference's gt_spec=None start no longer raises: store its own output")
            torch.manual_seed(_seed(name))
            x, t = torch.randn(shape), torch.full((B,), 0.0)
            cond, dt = inp["condition"].transpose(1, 2), 1.0 / c["steps"]
            step = flow.sample_euler if c["method"] == "euler" else flow.sample_rk4
            for _ in range(c["steps"]):
                x, t = step(x, t, dt, cond)
            out["out32"] = flow.denorm_spec(x.squeeze(1).transpose(1, 2)).numpy()
        else:
            out["out32"] = flow(inp["condition"], gt_spec=inp["gt_spec"], **kw).numpy()
    np.savez_compressed(path(name), **out)


def residual_ratios(model, name):
    """rms(layer update) / rms(layer input) of the oracle on a case's inputs (the weight scale's purpose)"""
    net, inp = build_oracle(model), build_inputs(name)
    ratios = []
    with torch.no_grad():
        x = torch.nn.functional.gelu(net.input_projection(torch.randn(inp["condition"].shape[0], MODELS[model]["mel"],
                                                                      inp["condition"].shape[1])))
        e = net.diffusion_embedding[0](torch.full((x.shape[0],), 500.0), torch.float32)
        for m in net.diffusion_embedding[1:]:
            e = m(e)
        for layer in net.residual_layers:
            y = layer(x, inp["condition"].transpose(1, 2), e.unsqueeze(-1))
            ratios.append(((y - x).pow(2).mean().sqrt() / x.pow(2).mean().sqrt()).item())
            x = y
    return ratios


def write_state_dict_keys():
    """reflow_state_dicts.json: [key, shape] of the reference's NaiveV2Diff (each model) and of Unit2Wav's
    reflow_model (RectifiedFlow around the w512 network)"""
    import json
    _, rf = _reference()
    sd = {m: [[k, list(v.shape)] for k, v in build_reference(m).state_dict().items()] for m in MODELS}
    sd["RectifiedFlow_w512"] = [[k, list(v.shape)] for k, v in rf.RectifiedFlow(build_reference("w512")).state_dict().items()]
    with open(os.path.join(HERE, "reflow_state_dicts.json"), "w") as f:
        json.dump(sd, f)


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    write_state_dict_keys()
    for model, case in (("w128", "reflow_w128_b1_t37_euler5_t07"), ("w512", "reflow_w512_b1_t24_euler3_t07")):
        print(model, "residual update / input per layer:", ["%.2f" % r for r in residual_ratios(model, case)])
    for n in names:
        generate(n)
        print("wrote", path(n))
