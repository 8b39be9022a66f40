"""Plain-torch restatement of the diffusion models' denoiser WaveNet (reference diffusion/wavenet.py) and of
GaussianDiffusion's inference samplers (diffusion/diffusion.py:216-384 with DPM-Solver++ and UniPC as it configures
them), on standard nn layers, usable in float64 (``.double()``), with the reference's state-dict keys and shapes.  The
samplers are written step by step as the methods define them (data predictions, differences, correctors), not as the
package's per-step linear combinations, so the two check each other.

TEST INFRASTRUCTURE ONLY.  tests/test_oracle_diffusion.py pins it to the reference's own outputs stored by
tests/golden/make_golden_diffusion.py; the GPU tests use it (float64, or fp32 eagerly on the GPU: what the reference runs
today) where the reference does not exist.  NaiveV2Diff's oracle is tests/reflow_oracle.VelocityNet.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from tests.reflow_oracle import StepEmbedding, seeded_weights  # noqa: F401  (seeded_weights: re-exported for the fixtures)


class ResidualBlock(nn.Module):
    def __init__(self, encoder_hidden, residual_channels):
        super().__init__()
        self.residual_channels = residual_channels
        self.dilated_conv = nn.Conv1d(residual_channels, 2 * residual_channels, 3, padding=1)
        self.diffusion_projection = nn.Linear(residual_channels, residual_channels)
        self.conditioner_projection = nn.Conv1d(encoder_hidden, 2 * residual_channels, 1)
        self.output_projection = nn.Conv1d(residual_channels, 2 * residual_channels, 1)

    def forward(self, x, cond, step):                        # x [B, C, T], step [B, C]
        y = self.dilated_conv(x + self.diffusion_projection(step)[:, :, None]) + self.conditioner_projection(cond)
        C = self.residual_channels
        y = self.output_projection(torch.sigmoid(y[:, :C]) * torch.tanh(y[:, C:]))
        return (x + y[:, :C]) / math.sqrt(2.0), y[:, C:]


class WaveNet(nn.Module):
    def __init__(self, in_dims=128, n_layers=20, n_chans=512, n_hidden=256):
        super().__init__()
        self.input_projection = nn.Conv1d(in_dims, n_chans, 1)
        self.diffusion_embedding = StepEmbedding(n_chans)
        self.mlp = nn.Sequential(nn.Linear(n_chans, n_chans * 4), nn.Mish(), nn.Linear(n_chans * 4, n_chans))
        self.residual_layers = nn.ModuleList([ResidualBlock(n_hidden, n_chans) for _ in range(n_layers)])
        self.skip_projection = nn.Conv1d(n_chans, n_chans, 1)
        self.output_projection = nn.Conv1d(n_chans, in_dims, 1)

    def forward(self, spec, diffusion_step, cond):
        """spec [B, 1, M, T], diffusion_step [B], cond [B, n_hidden, T] -> noise prediction [B, 1, M, T]"""
        dtype = self.input_projection.weight.dtype
        x = F.relu(self.input_projection(spec[:, 0].to(dtype)))
        step = self.mlp(self.diffusion_embedding(diffusion_step, dtype))
        cond = cond.to(dtype)
        skip = 0
        for layer in self.residual_layers:
            x, s = layer(x, cond, step)
            skip = skip + s
        x = F.relu(self.skip_projection(skip / math.sqrt(len(self.residual_layers))))
        return self.output_projection(x)[:, None]


def tables(timesteps=1000, max_beta=0.02):
    """the registered buffers of GaussianDiffusion (float64 numpy -> fp32), by name"""
    betas = np.linspace(1e-4, max_beta, timesteps)
    ac = np.cumprod(1.0 - betas)
    ac_prev = np.append(1.0, ac[:-1])
    var = betas * (1.0 - ac_prev) / (1.0 - ac)
    t = dict(betas=betas, alphas_cumprod=ac, sqrt_alphas_cumprod=np.sqrt(ac), sqrt_one_minus_alphas_cumprod=np.sqrt(1 - ac),
             sqrt_recip_alphas_cumprod=np.sqrt(1 / ac), sqrt_recipm1_alphas_cumprod=np.sqrt(1 / ac - 1),
             posterior_log_variance_clipped=np.log(np.maximum(var, 1e-20)),
             posterior_mean_coef1=betas * np.sqrt(ac_prev) / (1 - ac),
             posterior_mean_coef2=(1 - ac_prev) * np.sqrt(1 - betas) / (1 - ac))
    return {k: torch.tensor(v, dtype=torch.float32) for k, v in t.items()}


class Schedule:
    """the discrete VP schedule of betas[:t] as DPM-Solver / UniPC build it (fp32 tables), evaluated in float64"""

    def __init__(self, betas):
        la = 0.5 * torch.log(1 - betas).cumsum(0)
        lam = la - 0.5 * torch.log(1 - torch.exp(2 * la))
        cut = int((lam < -5.1).sum())                          # lambda decreases: the clipped tail
        la = la[:len(la) - cut]
        self.N = len(la)
        self.t = torch.linspace(0.0, 1.0, self.N + 1)[1:].double().numpy()
        self.la = la.double().numpy()

    def grid(self, steps):
        ts = torch.linspace(1.0, 1.0 / self.N, steps + 1)
        return ts.double().tolist(), ((ts - 1.0 / self.N) * self.N).tolist()

    def at(self, t):
        la = float(np.interp(t, self.t, self.la))
        sigma = math.sqrt(1 - math.exp(2 * la))
        return math.exp(la), sigma, la - math.log(sigma)


def sample(net, condition, noise, gt_spec, k_step, speedup, method, step_noise=None, k_step_max=1000, spec_min=-12,
           spec_max=2):
    """GaussianDiffusion.forward(infer=True) in the network's dtype, fed explicit noise: condition [B, T, M_cond],
    noise [B, 1, M, T] (the start's draw, in the start's layout), gt_spec [B, T, M] or None (then t = k_step_max),
    step_noise: DDPM's per-step draws [B, 1, M, T] in order -> [B, T, M].  Returns (mel, steps fed to the network)."""
    dtype = net.input_projection.weight.dtype
    tb = {k: v.double() for k, v in tables().items()}
    cond = condition.to(dtype).transpose(1, 2)
    B, dev = condition.shape[0], condition.device
    fed = []

    def eps(x, s):
        fed.append(float(s))
        return net(x, torch.full((B,), float(s), dtype=torch.float32, device=dev), cond)

    if gt_spec is None:
        t, x = k_step_max, noise.to(dtype)
    else:
        t = k_step
        norm = ((gt_spec.to(dtype) - spec_min) / (spec_max - spec_min) * 2 - 1).transpose(1, 2)[:, None]
        x = float(tb["sqrt_alphas_cumprod"][t - 1]) * norm + float(tb["sqrt_one_minus_alphas_cumprod"][t - 1]) * noise.to(dtype)
    ac = tb["alphas_cumprod"]
    if method is None or speedup == 1:
        for j, i in enumerate(reversed(range(t))):
            e = eps(x, i)
            x0 = float(tb["sqrt_recip_alphas_cumprod"][i]) * x - float(tb["sqrt_recipm1_alphas_cumprod"][i]) * e
            mean = float(tb["posterior_mean_coef1"][i]) * x0 + float(tb["posterior_mean_coef2"][i]) * x
            sd = math.exp(0.5 * float(tb["posterior_log_variance_clipped"][i])) if i else 0.0
            x = mean + sd * step_noise[j].to(dtype)
    elif method in ("dpm-solver", "unipc"):
        steps = t // speedup
        assert steps >= 2
        sch = Schedule(tables()["betas"][:t])
        ts, model_t = sch.grid(steps)
        al, sg, lm = zip(*(sch.at(v) for v in ts))
        pred = lambda x, k: (x - sg[k] * eps(x, model_t[k])) / al[k]
        ms = [pred(x, 0)]
        for k in range(1, steps + 1):
            h = lm[k] - lm[k - 1]
            phi = math.expm1(-h)
            base = sg[k] / sg[k - 1] * x - al[k] * phi * ms[-1]
            if method == "dpm-solver":
                order = 1 if k == 1 or (steps < 10 and k == steps) else 2
                x = base if order == 1 else base - 0.5 * al[k] * phi * (ms[-1] - ms[-2]) / ((lm[k - 1] - lm[k - 2]) / h)
                if k < steps:
                    ms.append(pred(x, k))
                continue
            # UniPC bh2: B(h) = expm1(-h); predictor of order min(2, history), corrector with the new data prediction
            Bh = math.expm1(-h)
            if k == steps:                                      # last step: first order, no corrector
                x = base
                break
            if k == 1:
                m_t = pred(base, k)
                x = base - al[k] * Bh * 0.5 * (m_t - ms[-1])
            else:
                r = (lm[k - 2] - lm[k - 1]) / h
                D1 = (ms[-2] - ms[-1]) / r
                m_t = pred(base - al[k] * Bh * 0.5 * D1, k)
                hh = -h
                hp = math.expm1(hh) / hh - 1
                b = torch.tensor([hp / Bh, 2 * (hp / hh - 0.5) / Bh], dtype=torch.float64)
                rho = torch.linalg.solve(torch.tensor([[1.0, 1.0], [r, 1.0]], dtype=torch.float64), b).tolist()
                x = base - al[k] * Bh * (rho[0] * D1 + rho[1] * (m_t - ms[-1]))
            ms.append(m_t)
    elif method in ("pndm", "ddim"):
        hist = []
        for i in reversed(range(0, t, speedup)):
            a_t, a_p = float(ac[i]), float(ac[max(i - speedup, 0)])
            e = eps(x, i)
            if method == "ddim":
                x = math.sqrt(a_p) * (x / math.sqrt(a_t) + (math.sqrt((1 - a_p) / a_p) - math.sqrt((1 - a_t) / a_t)) * e)
                continue

            def x_pred(x, n):
                return x + (a_p - a_t) * (x / (math.sqrt(a_t) * (math.sqrt(a_t) + math.sqrt(a_p))) -
                                          n / (math.sqrt(a_t) * (math.sqrt((1 - a_p) * a_t) + math.sqrt((1 - a_t) * a_p))))
            if not hist:
                e_prime = (e + eps(x_pred(x, e), max(i - speedup, 0))) / 2
            elif len(hist) == 1:
                e_prime = (3 * e - hist[-1]) / 2
            elif len(hist) == 2:
                e_prime = (23 * e - 16 * hist[-1] + 5 * hist[-2]) / 12
            else:
                e_prime = (55 * e - 59 * hist[-1] + 37 * hist[-2] - 9 * hist[-3]) / 24
            x = x_pred(x, e_prime)
            hist.append(e)
    else:
        raise NotImplementedError(method)
    return (x[:, 0].transpose(1, 2) + 1) / 2 * (spec_max - spec_min) + spec_min, fed
