"""Generate tests/golden/diffusion_grad_*.npz: the LIVE reference's diffusion training loss (diffusion/diffusion.py
GaussianDiffusion.forward with infer=False -> p_losses, loss_type 'l2') around its WaveNet (diffusion/wavenet.py) and
around NaiveV2Diff (diffusion/naive_v2_diff.py, as Unit2WavFast builds it), and its gradients, on the CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_diffusion_grad.py [case names; default: all]

The networks are make_golden_diffusion's seeded w64 WaveNet (3 layers) and its 2-layer w128 NaiveV2Diff ("naive"):
every weight non-zero -- the reference zero-initialises the output projection, which would make every inner gradient
vanish.  Weights are not stored.  Each file holds:

* the inputs ``condition`` [B, T, M_cond] and ``gt_spec`` [B, T, 128];
* the draws: ``t`` [B] (int64) and ``noise`` [B, T, 128], token-major -- the memory order of the reference's randn_like
  of the transposed [B, 1, M, T] view of norm_spec(gt_spec); ``t_max`` (-1 for the case with explicit t);
* ``loss32`` (the reference's forward under torch.manual_seed(seed)) and ``loss64`` (the reference's p_losses in
  float64 fed the same draws; its sinusoidal step embedding is handed the steps as float64, since an int64 step times
  the fp32 frequencies stays fp32 and the float64 MLP would refuse it);
* ``f64/<name>``: the float64 gradient of every parameter and of ``condition``, rounded to fp32, at the entries
  ``stored`` keeps (all of a tensor up to 2048 entries, else 2048 fixed random ones); ``err32/<name>``: the reference's
  own fp32 gradient's relative RMS error against it over the same entries; ``none``: the parameters whose gradient is
  None (NaiveV2Diff's unused LayerNorms).

The generator checks that replaying the stored draws through the reference's p_losses reproduces its seeded forward bit
for bit, which pins the draw order (torch.randint, then randn_like of the transposed view).  The case with explicit t
(0 and 999, the schedule's ends) calls p_losses directly.
"""
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

from tests.golden import make_golden_diffusion as mk  # noqa: E402
from tests.golden.make_golden_reflow_grad import rel_rms, sample_index  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = OrderedDict([
    ("diffusion_grad_w64_b1_t40_k100", dict(model="w64", B=1, T=40, k_step=100)),
    ("diffusion_grad_w64_b2_t33_k300", dict(model="w64", B=2, T=33, k_step=300)),
    ("diffusion_grad_w64_b3_t24_knone", dict(model="w64", B=3, T=24, k_step=None)),       # t_max = self.k_step = 1000
    ("diffusion_grad_w64_b2_t20_t0_999", dict(model="w64", B=2, T=20, t=[0, 999])),
    # every tap of the convolution's adjoint at an utterance edge
    ("diffusion_grad_w64_b2_t1_k100", dict(model="w64", B=2, T=1, k_step=100)),
    ("diffusion_grad_w64_b2_t2_k100", dict(model="w64", B=2, T=2, k_step=100)),
    ("diffusion_grad_w64_b3_t37_k100", dict(model="w64", B=3, T=37, k_step=100)),
    ("diffusion_grad_naive_b2_t30_k100", dict(model="naive", B=2, T=30, k_step=100)),
])


def path(name):
    return os.path.join(HERE, name + ".npz")


def _seed(name):
    return 5000 + list(CASES).index(name)


def t_max(name):
    c = CASES[name]
    return -1 if "t" in c else (1000 if c["k_step"] is None else c["k_step"])


def stored(name, grads):
    """{tensor name: the entries of its gradient that the fixture keeps}; they depend on the case and the name only"""
    order = sorted(grads)
    return OrderedDict((n, g.detach().reshape(-1).cpu()[sample_index(g.numel(), _seed(name) * 1000 + order.index(n))])
                       for n, g in grads.items() if g is not None)


def build_inputs(name):
    """condition [B, T, M_cond] and gt_spec [B, T, 128]: a ramp over the bins plus noise (log-mel-like)"""
    c = CASES[name]
    g = torch.Generator().manual_seed(_seed(name))
    Mc = mk.cond_channels(c["model"])
    ramp = lambda n: torch.linspace(-8.0, 0.5, n)[None, None, :]
    condition = ramp(Mc) + 1.5 * torch.randn(c["B"], c["T"], Mc, generator=g)
    gt = ramp(128) + 1.5 * torch.randn(c["B"], c["T"], 128, generator=g)
    return condition, gt


def reference_loss(gd, condition, gt, t, noise):
    """the reference's p_losses (its x_start from its norm_spec) fed the draws t [B], noise [B, T, M] token-major"""
    x0 = gd.norm_spec(gt).transpose(1, 2)[:, None, :, :]
    return gd.p_losses(x0, t, cond=condition.transpose(1, 2), noise=noise.transpose(1, 2)[:, None])


def generate(name):
    c = CASES[name]
    dd, _, _ = mk._reference()
    net = mk.build_reference(c["model"]).train()
    gd = dd.GaussianDiffusion(net, out_dims=128)
    condition, gt = build_inputs(name)
    B, T = c["B"], c["T"]
    cond32 = condition.clone().requires_grad_(True)
    torch.manual_seed(_seed(name))
    if "t" in c:
        t = torch.tensor(c["t"], dtype=torch.int64)
        noise = torch.empty_strided((B, 1, 128, T), (T * 128, T * 128, 1, 128)).normal_()[:, 0].transpose(1, 2)
        loss32 = reference_loss(gd, cond32, gt, t, noise)
    else:
        loss32 = gd(cond32, gt_spec=gt, infer=False, k_step=c["k_step"])
        # the same draws again, as the reference makes them: randint, then randn_like of the transposed view
        torch.manual_seed(_seed(name))
        t = torch.randint(0, t_max(name), (B,)).long()
        noise = torch.randn_like(gd.norm_spec(gt).transpose(1, 2)[:, None, :, :])[:, 0].transpose(1, 2)
        with torch.no_grad():
            replay = reference_loss(gd, condition, gt, t, noise)
        assert torch.equal(replay, loss32.detach()), (replay, loss32)
    loss32.backward()
    g32 = {n: p.grad for n, p in net.named_parameters()}
    g32["condition"] = cond32.grad
    net64 = copy.deepcopy(net).double()
    net64.zero_grad(set_to_none=True)
    for m in net64.modules():                   # int64 steps times fp32 frequencies stay fp32: take the steps in float64
        if type(m).__name__ in ("SinusoidalPosEmb", "DiffusionEmbedding"):
            m.forward = (lambda f: lambda x: f(x.double()))(m.forward)
    gd64 = dd.GaussianDiffusion(net64, out_dims=128).double()
    cond64 = condition.double().requires_grad_(True)
    loss64 = reference_loss(gd64, cond64, gt.double(), t, noise.double())
    loss64.backward()
    g64 = {n: p.grad for n, p in net64.named_parameters()}
    g64["condition"] = cond64.grad
    out = dict(condition=condition.numpy(), gt_spec=gt.numpy(), t=t.numpy(), noise=noise.contiguous().numpy(),
               t_max=np.array(t_max(name)), loss32=loss32.detach().numpy(), loss64=loss64.detach().numpy(),
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
