"""Generate tests/golden/reflow_grad_*.npz: the LIVE reference's reflow loss (reflow/reflow.py RectifiedFlow.forward
with infer=False -> reflow_loss, loss_type 'l2_lognorm') around its velocity network NaiveV2Diff (use_mlp=False, as
Unit2Wav builds it), and its gradients, on the CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_reflow_grad.py [case names; default: all]

The network is make_golden_reflow's w128 model (2 layers, seeded non-zero weights: the reference zero-initialises the
output projection, which would make every inner gradient vanish).  Weights are not stored.  Each file holds:

* the inputs ``condition`` [B, T, 128] and ``gt_spec`` [B, T, 128];
* the draws: ``t`` [B] (clipped) and ``x0`` [B, T, M], token-major -- the memory order of the reference's
  randn_like of the transposed [B, 1, M, T] view of norm(gt_spec);
* ``loss32`` (the reference's forward under torch.manual_seed(seed)) and ``loss64`` (the reference's reflow_loss in
  float64 fed the same draws);
* ``f64/<name>``: the float64 gradient of every parameter and of ``condition``, rounded to fp32, at the entries
  ``stored`` keeps (all of a tensor up to 2048 entries, else 2048 fixed random ones: the w128 model's gradients alone
  are 0.44 M floats, so each file stays near 200 KB); ``err32/<name>``: the reference's own fp32 gradient's relative
  RMS error against it over the same entries; ``none``: the parameters whose gradient is None (the layers' unused
  LayerNorms).

The generator checks that replaying the stored draws through the reference's reflow_loss reproduces its seeded forward
bit for bit, which pins the draw order (torch.rand, then randn_like of the transposed view).  The case with t at the
clip bounds calls reflow_loss with explicit t (0 and 1 clip to 1e-7 and 1 - 1e-7, whose fp32 weights underflow to 0).
"""
import contextlib
import copy
import json
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_golden_reflow as mk  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
MODEL = "w128"

CASES = OrderedDict([
    ("reflow_grad_w128_b1_t40_t0", dict(B=1, T=40, t_start=0.0)),
    ("reflow_grad_w128_b2_t33_t07", dict(B=2, T=33, t_start=0.7)),
    ("reflow_grad_w128_b3_t24_bounds", dict(B=3, T=24, t=[0.0, 0.97, 1.0])),
    # shorter than the depthwise convolution's 31-tap reach
    ("reflow_grad_w128_b1_t9_t07", dict(B=1, T=9, t_start=0.7)),
])


def path(name):
    return os.path.join(HERE, name + ".npz")


def _seed(name):
    return 3000 + list(CASES).index(name)


def sample_index(n, seed, k=2048):
    """indices of the stored entries of a flattened gradient of n elements (all of them up to k)"""
    if n <= k:
        return torch.arange(n)
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:k].sort().values


def stored(name, grads):
    """{tensor name: the entries of its gradient that the fixture keeps}; the entries of a tensor depend on the case
    and the tensor's name only"""
    order = sorted(grads)
    return OrderedDict((n, g.detach().reshape(-1).cpu()[sample_index(g.numel(), _seed(name) * 1000 + order.index(n))])
                       for n, g in grads.items() if g is not None)


def build_inputs(name):
    """condition [B, T, 128] and gt_spec [B, T, 128]: a ramp over the bins plus noise (log-mel-like)"""
    c, m = CASES[name], mk.MODELS[MODEL]
    g = torch.Generator().manual_seed(_seed(name))
    ramp = torch.linspace(-8.0, 0.5, m["cond"])[None, None, :]
    condition = ramp + 1.5 * torch.randn(c["B"], c["T"], m["cond"], generator=g)
    gt = ramp[..., :m["mel"]] + 1.5 * torch.randn(c["B"], c["T"], m["mel"], generator=g)
    return condition, gt


def draws(B, T, M, t_start):
    """the reference's draws in its order, fp32 on the CPU: t, then x_0 [B, T, M] token-major"""
    t = t_start + (1.0 - t_start) * torch.rand(B)
    t = torch.clip(t, 1e-7, 1 - 1e-7)
    x0 = torch.empty_strided((B, 1, M, T), (T * M, T * M, 1, M)).normal_()
    return t, x0[:, 0].transpose(1, 2)


def oracle_loss(net, condition, gt, t, x0, spec_min=-12, spec_max=2):
    """the reflow loss ('l2_lognorm') around tests/reflow_oracle.VelocityNet in the network's dtype, fed explicit draws:
    condition [B, T, M_cond], gt [B, T, M], t [B], x0 [B, T, M] token-major -> loss []"""
    dtype = net.input_projection.weight.dtype
    x1 = ((gt.to(dtype) - spec_min) / (spec_max - spec_min) * 2 - 1).transpose(1, 2)[:, None]
    x0 = x0.to(dtype).transpose(1, 2)[:, None]
    t = t.to(dtype)
    xt = x0 + t[:, None, None, None] * (x1 - x0)
    v = net(xt, 1000 * t, condition.to(dtype).transpose(1, 2))
    w = 0.398942 / t / (1 - t) * torch.exp(-0.5 * torch.log(t / (1 - t)) ** 2)
    return torch.mean(w[:, None, None, None] * (x1 - x0 - v) ** 2)


@contextlib.contextmanager
def _fixed_randn_like(x0):
    """torch.randn_like returns x0 [B, T, M] in the argument's [B, 1, M, T] layout and dtype"""
    orig = torch.randn_like
    torch.randn_like = lambda x, **kw: x0.to(x.dtype).transpose(1, 2)[:, None].clone()
    try:
        yield
    finally:
        torch.randn_like = orig


def reference_loss(flow, condition, gt, t, x0):
    """the reference's reflow_loss (its x_1 from its norm_spec) fed the draws t, x0"""
    x1 = flow.norm_spec(gt).transpose(1, 2)[:, None, :, :]
    with _fixed_randn_like(x0):
        return flow.reflow_loss(x1, t, cond=condition.transpose(1, 2))


def rel_rms(a, b):
    a, b = a.double(), b.double()
    return float((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-300))


def generate(name):
    c = CASES[name]
    _, rf = mk._reference()
    M = mk.MODELS[MODEL]["mel"]
    net = mk.build_reference(MODEL).train()
    flow = rf.RectifiedFlow(net, out_dims=M)
    condition, gt = build_inputs(name)
    B, T = c["B"], c["T"]
    cond32 = condition.clone().requires_grad_(True)
    torch.manual_seed(_seed(name))
    if "t" in c:
        t, x0 = torch.clip(torch.tensor(c["t"]), 1e-7, 1 - 1e-7), draws(B, T, M, 0.0)[1]
        loss32 = reference_loss(flow, cond32, gt, t, x0)
    else:
        loss32 = flow(cond32, gt_spec=gt, infer=False, t_start=c["t_start"])
        torch.manual_seed(_seed(name))
        t, x0 = draws(B, T, M, c["t_start"])
        with torch.no_grad():
            replay = reference_loss(flow, condition, gt, t, x0)
        assert torch.equal(replay, loss32.detach()), (replay, loss32)
    loss32.backward()
    g32 = {n: p.grad for n, p in net.named_parameters()}
    g32["condition"] = cond32.grad
    net64 = copy.deepcopy(net).double()
    net64.zero_grad(set_to_none=True)
    flow64 = rf.RectifiedFlow(net64, out_dims=M)
    cond64 = condition.double().requires_grad_(True)
    loss64 = reference_loss(flow64, cond64, gt.double(), t.double(), x0.double())
    loss64.backward()
    g64 = {n: p.grad for n, p in net64.named_parameters()}
    g64["condition"] = cond64.grad
    out = dict(condition=condition.numpy(), gt_spec=gt.numpy(), t=t.numpy(), x0=x0.contiguous().numpy(),
               loss32=loss32.detach().numpy(), loss64=loss64.detach().numpy(),
               none=np.array(json.dumps(sorted(n for n, v in g64.items() if v is None))))
    s32 = stored(name, g32)
    for n, v in stored(name, g64).items():
        out["f64/" + n] = v.float().numpy()
        out["err32/" + n] = np.array(rel_rms(s32[n], v))
    np.savez_compressed(path(name), **out)


if __name__ == "__main__":
    for n in sys.argv[1:] or list(CASES):
        generate(n)
        print("wrote", path(n), "%.2f MB" % (os.path.getsize(path(n)) / 2 ** 20))
