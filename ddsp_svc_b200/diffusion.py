"""The diffusion models' sampler on the GPU: the WaveNet denoiser (reference diffusion/wavenet.py) and GaussianDiffusion
(diffusion/diffusion.py) with its five samplers -- DPM-Solver++, UniPC, PNDM, DDIM and DDPM -- inference only.

Same constructors, parameter trees and registered buffers as the reference, so a Unit2Mel / Unit2Wav / Unit2WavFast
checkpoint's ``decoder.*`` / ``diff_model.*`` keys load strictly.  ``GaussianDiffusion`` takes as ``denoise_fn`` this
module's ``WaveNet`` or the package's ``NaiveV2Diff`` (what Unit2WavFast builds); both give the sampler the same three
operations: ``_cond_rows`` (every layer's condition projection, once per call), ``_step_rows`` (the step embedding, its
MLP and every layer's step projection for every evaluation of the call, batched: every schedule below is known on the
host before the loop starts) and ``_velocity`` (one evaluation from a GEMM operand, without the output bias).

Execution: activations stay token-major [B, T, C].  Per WaveNet evaluation: the input-projection GEMM; per layer the
k = 3 convolution as ONE GEMM over a [B T, 3 C] operand (the three taps side by side, zero outside each utterance), the
gate, the output-projection GEMM and the residual / skip update; the skip-projection and output-projection GEMMs.  The
stages between the GEMMs are the kernels of csrc/diffusion.cu, which write the next GEMM's operand directly.  The sampler
is one loop over the evaluations: after each, ONE df_update kernel adds the output bias and forms the next point as a
linear combination of the current point, the network output and at most three stored tensors, with per-step
coefficients computed on the host (float64 from the reference's fp32 schedule tables, rounded to fp32 once).  The start
is csrc/reflow.cu's rf_start (q_sample has its formula), the finish rf_finish (denorm_spec).  The GEMMs run at
``gemm_precision`` (unit2control._Gemm: "3xtf32" default, "fp32", "tf32").

Reference behaviour kept on purpose (DESIGN.md section 4.15): the shallow start noises to step k_step - 1 while DDIM and
PNDM first denoise at k_step - speedup; the start's noise is randn_like of the transposed [B, 1, M, T] view, which fills
[B, T, M] in memory order.  Where the reference cannot run what its code means, the meaning runs: its PNDM takes
``max(t - interval, 0)`` of a [B] tensor, which raises for B > 1 (and hands the network a Python int when the step is
clipped to 0); here every B runs with the step clipped at 0.

Training (infer=False, p_losses) is not built: it and every call under grad raise NotImplementedError.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from .ops import _need_cuda_f32, _stream
from .reflow import NaiveV2Diff, _DiffusionEmbedding, _under_grad
from .unit2control import _Gemm, _k, _split

_NO_TRAINING = ("%s: training (p_losses and the denoiser's gradients) is not built; run inference with infer=True under "
                "torch.no_grad()")


class _ResidualBlock(nn.Module):                 # wavenet.py:31-62 (dilation 1 in every configuration)
    def __init__(self, encoder_hidden, residual_channels, dilation):
        super().__init__()
        self.residual_channels = residual_channels
        self.dilated_conv = nn.Conv1d(residual_channels, 2 * residual_channels, kernel_size=3, padding=dilation,
                                      dilation=dilation)
        self.diffusion_projection = nn.Linear(residual_channels, residual_channels)
        self.conditioner_projection = nn.Conv1d(encoder_hidden, 2 * residual_channels, 1)
        self.output_projection = nn.Conv1d(residual_channels, 2 * residual_channels, 1)


class WaveNet(nn.Module):
    #: precision of the library GEMMs, see unit2control._Gemm: "3xtf32" (default), "fp32", "tf32"
    gemm_precision = "3xtf32"

    def __init__(self, in_dims=128, n_layers=20, n_chans=384, n_hidden=256):
        super().__init__()
        unsupported = [name for name, bad in (("n_chans=%r (not a multiple of 64)" % (n_chans,), n_chans <= 0 or n_chans % 64),
                                              ("n_layers=%r" % (n_layers,), n_layers < 1),
                                              ("in_dims=%r" % (in_dims,), in_dims < 1),
                                              ("n_hidden=%r" % (n_hidden,), n_hidden < 1)) if bad]
        if unsupported:
            raise NotImplementedError("WaveNet: n_chans must be a positive multiple of 64 and the other sizes positive "
                                      "(every configuration builds n_chans 512); got " + ", ".join(unsupported))
        self.input_projection = nn.Conv1d(in_dims, n_chans, 1)
        nn.init.kaiming_normal_(self.input_projection.weight)
        self.diffusion_embedding = _DiffusionEmbedding(n_chans)
        self.mlp = nn.Sequential(nn.Linear(n_chans, n_chans * 4), nn.Mish(), nn.Linear(n_chans * 4, n_chans))
        self.residual_layers = nn.ModuleList([_ResidualBlock(n_hidden, n_chans, 1) for _ in range(n_layers)])
        self.skip_projection = nn.Conv1d(n_chans, n_chans, 1)
        nn.init.kaiming_normal_(self.skip_projection.weight)
        self.output_projection = nn.Conv1d(n_chans, in_dims, 1)
        nn.init.zeros_(self.output_projection.weight)
        self.mel_channels, self.condition_dim, self.dim = in_dims, n_hidden, n_chans
        self.__dict__["_packed"] = None

    # ---- weights in the layouts the GEMMs want, rebuilt when a parameter changes (load_state_dict, .to) ----
    def _pack(self):
        key = (self.gemm_precision,) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        c = self.__dict__.get("_packed")
        if c is not None and c[0] == key:
            return c[1]
        d = lambda t: t.detach().contiguous()
        w2 = lambda conv: conv.weight.detach()[:, :, 0].contiguous()
        layers = self.residual_layers
        P = dict(in_w=w2(self.input_projection), in_b=d(self.input_projection.bias),
                 mlp1_w=d(self.mlp[0].weight), mlp1_b=d(self.mlp[0].bias), mlp2_w=d(self.mlp[2].weight),
                 mlp2_b=d(self.mlp[2].bias),
                 step_w=torch.cat([d(Ly.diffusion_projection.weight) for Ly in layers]),
                 step_b=torch.cat([d(Ly.diffusion_projection.bias) for Ly in layers]),
                 # the convolution's bias rides with the condition projection: z = conv(y) + (cond_proj(c) + both biases)
                 cond_w=torch.cat([w2(Ly.conditioner_projection) for Ly in layers]),
                 cond_b=torch.cat([d(Ly.conditioner_projection.bias + Ly.dilated_conv.bias) for Ly in layers]),
                 skip_w=w2(self.skip_projection), skip_b=d(self.skip_projection.bias),
                 out_w=w2(self.output_projection), out_b=d(self.output_projection.bias))
        # conv weight [2C, C, 3] -> [2C, 3C]: column block k multiplies the operand's block k, y(t + k - 1)
        P["layers"] = [dict(conv_w=Ly.dilated_conv.weight.detach().permute(0, 2, 1).reshape(2 * self.dim, 3 * self.dim)
                            .contiguous(), out_w=w2(Ly.output_projection), out_b=d(Ly.output_projection.bias))
                       for Ly in layers]
        if self.gemm_precision == "3xtf32":          # weights of every GEMM as TF32-exact (hi, lo) pairs, once per checkpoint
            for dd in [P] + P["layers"]:
                for name in [n for n in dd if n.endswith("_w")]:
                    dd[name] = _split(dd[name])
        self.__dict__["_packed"] = (key, P)
        return P

    # ---- the sampler's three operations (the same names and signatures as NaiveV2Diff's) ----
    def _step_rows(self, g, P, steps):
        """diffusion steps [E] -> every layer's step projection [E, n_layers C] (embedding, MLP, projections)"""
        e1 = g.linear(self.diffusion_embedding(steps), P["mlp1_w"], P["mlp1_b"])
        e2 = g.linear(F.mish(e1), P["mlp2_w"], P["mlp2_b"])
        return g.linear(e2, P["step_w"], P["step_b"])

    def _cond_rows(self, g, P, cond_tm):
        """condition [B, T, n_hidden] token-major -> every layer's condition projection plus both biases
        [B T, n_layers 2 C] (one GEMM)"""
        return g.mm(g.split(cond_tm.reshape(-1, cond_tm.shape[-1])), P["cond_w"], P["cond_b"])

    _operand = staticmethod(NaiveV2Diff._operand)
    _ptrs = staticmethod(NaiveV2Diff._ptrs)

    def _velocity(self, g, P, xs, steps, step_stride, conds, B, T, out_bias=None):
        """one evaluation of the denoiser: xs the input operand [B T, M] -> output projection [B T, M] (+ out_bias);
        steps: the step rows of this evaluation ([B or 1, n_layers C] from row stride step_stride), conds
        [B T, n_layers 2 C]"""
        L, C, dev, N, nL = _lib.lib(), self.dim, conds.device, B * T, len(P["layers"])
        new = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        h, skip = new(N, C), new(N, C)
        us, vs = self._operand(g, N, 3 * C, dev), self._operand(g, N, C, dev)
        (uh, ul), (vh, vl) = self._ptrs(us), self._ptrs(vs)
        G = g.mm(xs, P["in_w"])
        _k(L.b2d_df_layer(G.data_ptr(), P["in_b"].data_ptr(), h.data_ptr(), 0, 0, steps.data_ptr(), step_stride, 1.0, B, T,
                          C, uh, ul, _stream()), "b2d_df_layer")
        skip_div = math.sqrt(nL)
        for i, Ly in enumerate(P["layers"]):
            Z = g.mm(us, Ly["conv_w"])                                                   # [B T, 2 C]
            _k(L.b2d_df_gate(Z.data_ptr(), conds.data_ptr() + 4 * i * 2 * C, conds.shape[1], N, C, vh, vl, _stream()),
               "b2d_df_gate")
            R = g.mm(vs, Ly["out_w"])                                                    # [B T, 2 C]: residual | skip
            last = i + 1 == nL
            sp = 0 if last else steps.data_ptr() + 4 * (i + 1) * C
            oh, ol = (vh, vl) if last else (uh, ul)
            _k(L.b2d_df_layer(R.data_ptr(), Ly["out_b"].data_ptr(), h.data_ptr(), skip.data_ptr(), 1 if i == 0 else 2, sp,
                              step_stride, skip_div, B, T, C, oh, ol, _stream()), "b2d_df_layer")
        S = g.mm(vs, P["skip_w"])
        _k(L.b2d_df_relu(S.data_ptr(), P["skip_b"].data_ptr(), N, C, vh, vl, _stream()), "b2d_df_relu")
        return g.mm(vs, P["out_w"], out_bias)

    def forward(self, spec, diffusion_step, cond):
        """spec [B, 1, M, T] or [B, M, T], diffusion_step [B] (or one value for every utterance), cond [B, n_hidden, T]
        -> the predicted noise [B, 1, M, T] (wavenet.py:84-108)"""
        if _under_grad(self, spec, diffusion_step, cond):
            raise NotImplementedError(_NO_TRAINING % "WaveNet")
        x = spec[:, 0] if spec.dim() == 4 else spec
        _need_cuda_f32("spec", x)
        _need_cuda_f32("cond", cond)
        B, M, T = x.shape
        if M != self.mel_channels or cond.shape != (B, self.condition_dim, T):
            raise ValueError("WaveNet: spec [B, 1, %d, T] and cond [B, %d, T] expected, got %s and %s"
                             % (self.mel_channels, self.condition_dim, tuple(spec.shape), tuple(cond.shape)))
        steps = torch.as_tensor(diffusion_step, device=x.device).reshape(-1).expand(B)
        with torch.no_grad(), _Gemm(self.gemm_precision) as g:
            P = self._pack()
            srows = self._step_rows(g, P, steps).contiguous()
            crows = self._cond_rows(g, P, cond.transpose(1, 2).contiguous())
            xs = self._operand(g, B * T, M, x.device)
            hi, lo = self._ptrs(xs)
            _k(_lib.lib().b2d_rf_start(x.contiguous().data_ptr(), 0, 0.0, 1.0, 0.0, 1.0, B, T, M, 0, hi, lo, _stream()),
               "b2d_rf_start")
            v = self._velocity(g, P, xs, srows, srows.shape[1], crows, B, T, out_bias=P["out_b"])
        return v.reshape(B, T, M).transpose(1, 2).contiguous()[:, None]


# ---- the samplers' schedules and coefficients (host, float64 from the reference's fp32 tables) -----------------------------
def _vp_schedule(betas):
    """the discrete VP schedule DPM-Solver and UniPC build from betas[:t] (fp32, as the reference computes it):
    log alpha_n = 1/2 sum_{i <= n} log(1 - beta_i), with the tail where the half log-SNR falls below -5.1 dropped, on the
    times (n + 1) / N.  -> (log alpha [N], times [N], N) as fp32 tensors"""
    log_alpha = 0.5 * torch.log(1 - betas).cumsum(dim=0)
    lam = log_alpha - 0.5 * torch.log(1.0 - torch.exp(2.0 * log_alpha))
    drop = int(torch.searchsorted(torch.flip(lam, [0]), torch.tensor(-5.1)))
    if drop > 0:
        log_alpha = log_alpha[:-drop]
    n = log_alpha.shape[0]
    return log_alpha, torch.linspace(0.0, 1.0, n + 1)[1:], n


class _Marginals:
    """alpha, sigma and the half log-SNR lambda at continuous times, by linear interpolation of log alpha between the
    schedule's knots (the outer segments extended), in float64"""

    def __init__(self, log_alpha, times):
        self.la, self.ts = log_alpha.double().numpy(), times.double().numpy()

    def __call__(self, t):
        i = int(np.clip(np.searchsorted(self.ts, t) - 1, 0, len(self.ts) - 2))
        la = self.la[i] + (t - self.ts[i]) * (self.la[i + 1] - self.la[i]) / (self.ts[i + 1] - self.ts[i])
        sigma = math.sqrt(-math.expm1(2.0 * la))
        return math.exp(la), sigma, la - math.log(sigma)


class _Eval:
    """one network evaluation of a sampler and the df_update after it: the step value fed to the network, the eight
    coefficients, the history slots read as h1..h3 (None: not read), the slot that receives d (None: d not kept),
    whether x is stored, whether a fresh noise tensor is drawn and whether the next operand is written"""
    __slots__ = ("step", "coef", "reads", "write", "store", "noise", "emit")

    def __init__(self, step, coef, reads=(None, None, None), write=None, store=True, noise=False, emit=True):
        self.step, self.coef, self.reads, self.write = float(step), coef, reads, write
        self.store, self.noise, self.emit = store, noise, emit


def _coef(a_x=0.0, a_e=1.0, c_x=0.0, c_d=0.0, c_1=0.0, c_2=0.0, c_3=0.0, c_n=0.0):
    return [a_x, a_e, c_x, c_d, c_1, c_2, c_3, c_n]


def _multistep_plan(betas, steps, method):
    """DPM-Solver++ (multistep, order 2, lower-order final step when steps < 10) or UniPC (variant bh2, multistep, order
    2, first-order last step, a corrector after every step but the last) from t = 1 to 1/N on the uniform time grid,
    the model fed (t - 1/N) N.  The kernel's x is the point the network saw; d = the data prediction
    x0 = (x - sigma eps) / alpha; history: the previous data predictions."""
    log_alpha, times, n = _vp_schedule(betas)
    grid = torch.linspace(1.0, 1.0 / n, steps + 1)                      # fp32, as the reference's get_time_steps
    model_t = ((grid - 1.0 / n) * n).tolist()                           # fp32 arithmetic, then exact in float64
    mg = _Marginals(log_alpha, times)
    al, sg, lm = zip(*(mg(float(t)) for t in grid.double()))
    plan = []
    for e in range(steps):
        k = e + 1                                                        # the step this evaluation's update completes
        a_x, a_e = 1.0 / al[e], -sg[e] / al[e]
        h = lm[k] - lm[k - 1]
        phi = math.expm1(-h)
        S, Q = sg[k] / sg[k - 1], -al[k] * phi
        if method == "dpm-solver":
            order = 1 if e == 0 or (steps < 10 and k == steps) else 2
            if order == 1:
                coef = _coef(a_x, a_e, S, Q)
            else:
                r0 = (lm[k - 1] - lm[k - 2]) / h
                coef = _coef(a_x, a_e, S, Q + 0.5 * Q / r0, -0.5 * Q / r0)
            plan.append(_Eval(model_t[e], coef, (0 if order == 2 else None, None, None), 0 if k < steps else None,
                              emit=k < steps))
            continue
        # UniPC: this evaluation is at the point predicted for step e (e >= 1); x_e = p_e + cm_e m_e + cm_1 m_{e-1} +
        # cm_2 m_{e-2} is its corrected value, then the predictor of step k = e + 1 (or the final first-order step)
        cm_e = cm_1 = cm_2 = 0.0
        if e >= 1:
            he = lm[e] - lm[e - 1]
            A = al[e] * math.expm1(-he)                                  # alpha B(h), B(h) = expm1(-h) for bh2
            if e == 1:
                cm_e, cm_1 = -0.5 * A, 0.5 * A
            else:
                re = (lm[e - 2] - lm[e - 1]) / he
                hh = -he
                hp = math.expm1(hh) / hh - 1.0
                b1 = hp / math.expm1(hh)
                b2 = 2.0 * (hp / hh - 0.5) / math.expm1(hh)
                rho1 = (b2 - re * b1) / (1.0 - re)                       # [[1, 1], [re, 1]] rho = [b1, b2]
                rho0 = b1 - rho1
                cm_e = -A * rho1
                cm_1 = A * (rho1 - (0.5 - rho0) / re)
                cm_2 = A * (0.5 - rho0) / re
        pred = 0.0
        if 2 <= k < steps:                                               # second-order predictor of step k
            pred = al[k] * math.expm1(-h) * 0.5 / ((lm[k - 2] - lm[k - 1]) / h)
        coef = _coef(a_x, a_e, S, S * cm_e + Q + pred, S * cm_1 - pred, S * cm_2)
        plan.append(_Eval(model_t[e], coef, ((e - 1) % 2 if e >= 1 else None, e % 2 if e >= 2 else None, None),
                          e % 2 if k < steps else None, emit=k < steps))
    return plan, 1 if method == "dpm-solver" else 2


def _discrete_plan(buf, t, speedup, method):
    """PNDM, DDIM (steps t - speedup, t - 2 speedup, ..., down to the first multiple below t) and DDPM (every step
    t - 1 ... 0) from the registered fp32 buffers.  PNDM's first step evaluates twice; its history is the last three
    noise predictions (d = eps)."""
    ac = buf["alphas_cumprod"].double().numpy()
    plan = []
    if method == "ddpm":
        sra, srm = buf["sqrt_recip_alphas_cumprod"].double().numpy(), buf["sqrt_recipm1_alphas_cumprod"].double().numpy()
        c1, c2 = buf["posterior_mean_coef1"].double().numpy(), buf["posterior_mean_coef2"].double().numpy()
        lv = buf["posterior_log_variance_clipped"].double().numpy()
        for i in reversed(range(t)):
            sd = math.exp(0.5 * lv[i]) if i != 0 else 0.0
            plan.append(_Eval(i, _coef(sra[i], -srm[i], c2[i], c1[i], c_n=sd), noise=True, emit=i > 0))
        return plan, 0
    seq = list(reversed(range(0, t, speedup)))
    for j, i in enumerate(seq):
        a_t, a_p = ac[i], ac[max(i - speedup, 0)]
        last = j + 1 == len(seq)
        if method == "ddim":
            c_x = math.sqrt(a_p) / math.sqrt(a_t)
            c_e = math.sqrt(a_p) * (math.sqrt((1 - a_p) / a_p) - math.sqrt((1 - a_t) / a_t))
            plan.append(_Eval(i, _coef(c_x=c_x, c_d=c_e), emit=not last))
            continue
        # PNDM: x' = p x + q e' (get_x_pred) with e' the linear multistep combination of the noise predictions
        sa, sp = math.sqrt(a_t), math.sqrt(a_p)
        p = 1.0 + (a_p - a_t) / (sa * (sa + sp))
        q = -(a_p - a_t) / (sa * (math.sqrt((1 - a_p) * a_t) + math.sqrt((1 - a_t) * a_p)))
        if j == 0:
            plan.append(_Eval(i, _coef(c_x=p, c_d=q), write=0, store=False))                   # operand of x_pred only
            plan.append(_Eval(max(i - speedup, 0), _coef(c_x=p, c_d=0.5 * q, c_1=0.5 * q), (0, None, None),
                              emit=not last))
            continue
        w = {1: (3, -1, 0, 0, 2), 2: (23, -16, 5, 0, 12), 3: (55, -59, 37, -9, 24)}[min(j, 3)]
        reads = tuple((j - k) % 3 if k <= min(j, 3) else None for k in (1, 2, 3))
        plan.append(_Eval(i, _coef(c_x=p, c_d=q * w[0] / w[4], c_1=q * w[1] / w[4], c_2=q * w[2] / w[4],
                                   c_3=q * w[3] / w[4]), reads, j % 3, emit=not last))
    return plan, 3 if method == "pndm" else 0


_BUFFERS = ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod",
            "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_variance",
            "posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2", "spec_min", "spec_max")


class GaussianDiffusion(nn.Module):
    def __init__(self, denoise_fn, out_dims=128, timesteps=1000, k_step=1000, max_beta=0.02, spec_min=-12, spec_max=2):
        super().__init__()
        if not isinstance(denoise_fn, (WaveNet, NaiveV2Diff)):
            raise ValueError("GaussianDiffusion: denoise_fn must be ddsp_svc_b200.WaveNet or ddsp_svc_b200.NaiveV2Diff, "
                             "got %s" % type(denoise_fn).__name__)
        self.denoise_fn = denoise_fn
        self.out_dims = out_dims
        # diffusion.py:73-110: the linear beta schedule and the DDPM tables, float64, stored as fp32 buffers
        betas = np.linspace(1e-4, max_beta, timesteps)
        alphas = 1.0 - betas
        ac = np.cumprod(alphas, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        self.num_timesteps = int(betas.shape[0])
        self.k_step = k_step
        post_var = betas * (1.0 - ac_prev) / (1.0 - ac)
        tables = dict(betas=betas, alphas_cumprod=ac, alphas_cumprod_prev=ac_prev, sqrt_alphas_cumprod=np.sqrt(ac),
                      sqrt_one_minus_alphas_cumprod=np.sqrt(1.0 - ac), log_one_minus_alphas_cumprod=np.log(1.0 - ac),
                      sqrt_recip_alphas_cumprod=np.sqrt(1.0 / ac), sqrt_recipm1_alphas_cumprod=np.sqrt(1.0 / ac - 1),
                      posterior_variance=post_var,
                      posterior_log_variance_clipped=np.log(np.maximum(post_var, 1e-20)),
                      posterior_mean_coef1=betas * np.sqrt(ac_prev) / (1.0 - ac),
                      posterior_mean_coef2=(1.0 - ac_prev) * np.sqrt(alphas) / (1.0 - ac))
        for name, v in tables.items():
            self.register_buffer(name, torch.tensor(v, dtype=torch.float32))
        self.register_buffer("spec_min", torch.FloatTensor([spec_min])[None, None, :out_dims])
        self.register_buffer("spec_max", torch.FloatTensor([spec_max])[None, None, :out_dims])
        self.__dict__["_host_tables"] = None

    def _host(self):
        """the buffers as CPU fp32 tensors, copied once per change (load_state_dict, .to)"""
        key = tuple((b.data_ptr(), b._version) for b in (getattr(self, n) for n in _BUFFERS))
        c = self.__dict__.get("_host_tables")
        if c is None or c[0] != key:
            c = (key, {n: getattr(self, n).detach().cpu().reshape(-1) for n in _BUFFERS})
            self.__dict__["_host_tables"] = c
        return c[1]

    def norm_spec(self, x):
        return (x - self.spec_min) / (self.spec_max - self.spec_min) * 2 - 1

    def denorm_spec(self, x):
        return (x + 1) / 2 * (self.spec_max - self.spec_min) + self.spec_min

    def forward(self, condition, gt_spec=None, infer=True, infer_speedup=10, method='dpm-solver', k_step=None,
                use_tqdm=True):
        """condition [B, T, M_cond] -> the sampled mel [B, T, M] (diffusion.py:216-378).  The start: gt_spec or k_step
        None -> ONE torch.randn((B, 1, M, T)) from t = self.k_step; otherwise q_sample(norm(gt_spec), k_step - 1) with
        its noise drawn as randn_like of the transposed [B, 1, M, T] view, from t = k_step.  Then ``method``:
        'dpm-solver', 'unipc' (t // infer_speedup steps, at least 2), 'pndm', 'ddim'; None or infer_speedup 1: DDPM,
        one torch.randn((B, 1, M, T)) per step.  The draws happen on condition's device in the reference's order, so
        seeded runs compare.  ``use_tqdm`` is accepted and ignored."""
        if not infer:
            raise NotImplementedError(_NO_TRAINING % "GaussianDiffusion")
        if _under_grad(self, condition, gt_spec):
            raise NotImplementedError(_NO_TRAINING % "GaussianDiffusion")
        _need_cuda_f32("condition", condition)
        fn, M, dev = self.denoise_fn, self.out_dims, condition.device
        B, T, Mc = condition.shape
        if M != fn.mel_channels or Mc != fn.condition_dim:
            raise ValueError("GaussianDiffusion: out_dims / condition width do not match the denoiser")
        if gt_spec is None or k_step is None:
            t, gt = self.k_step, None
            noise = torch.randn((B, 1, M, T), device=dev)
        else:
            _need_cuda_f32("gt_spec", gt_spec)
            if gt_spec.shape != (B, T, M):
                raise ValueError("GaussianDiffusion: gt_spec must be [B, T, %d] like condition" % M)
            t, gt = int(k_step), gt_spec.contiguous()
            # randn_like(x_start) of the transposed view keeps its strides: the draw fills [B, T, M] in order
            noise = torch.empty_strided((B, 1, M, T), (T * M, T * M, 1, M), device=dev).normal_()
        return self._sample(condition, noise, gt, t, infer_speedup, method)

    def _sample(self, condition, noise, gt_spec, t, infer_speedup, method, step_noise=None):
        """forward after the start's draw: noise [B, 1, M, T] (any strides), gt_spec [B, T, M] or None, t the first
        step (k_step, or self.k_step without gt_spec).  DDPM draws its per-step noise here, one torch.randn((B, 1, M, T))
        per step, or takes them from ``step_noise`` (an iterable of [B, 1, M, T] tensors) when given."""
        fn, M, dev = self.denoise_fn, self.out_dims, condition.device
        B, T, _ = condition.shape
        if t < 1:
            raise ValueError("GaussianDiffusion: the first step (k_step) must be a positive int, got %r" % (t,))
        buf = self._host()
        if method is None or infer_speedup <= 1:
            plan, slots = _discrete_plan(buf, t, 1, "ddpm")
        elif method in ("dpm-solver", "unipc"):
            steps = t // infer_speedup
            if steps < 2:
                raise ValueError("GaussianDiffusion: %s needs at least 2 steps (order 2), got k_step // infer_speedup = %d"
                                 % (method, steps))
            plan, slots = _multistep_plan(buf["betas"][:t], steps, method)
        elif method in ("pndm", "ddim"):
            plan, slots = _discrete_plan(buf, t, infer_speedup, method)
        else:
            raise NotImplementedError(method)
        L, N = _lib.lib(), B * T
        spec_min = float(buf["spec_min"][0])
        spec_range = float(buf["spec_max"][0] - buf["spec_min"][0])
        if gt_spec is None:
            ts, one_m = 0.0, 1.0
        else:
            ts, one_m = float(buf["sqrt_alphas_cumprod"][t - 1]), float(buf["sqrt_one_minus_alphas_cumprod"][t - 1])
        noise = noise[:, 0].contiguous()                                   # channel-major [B, M, T] for rf_start
        with torch.no_grad(), _Gemm(fn.gemm_precision) as g:
            P = fn._pack()
            crows = fn._cond_rows(g, P, condition.contiguous())
            srows = fn._step_rows(g, P, torch.tensor([ev.step for ev in plan], dtype=torch.float32).to(dev)).contiguous()
            coefs = torch.tensor([ev.coef for ev in plan], dtype=torch.float32).to(dev)
            x = torch.empty(N, M, dtype=torch.float32, device=dev)
            hist = [torch.empty(N, M, dtype=torch.float32, device=dev) for _ in range(slots)]
            xs = fn._operand(g, N, M, dev)
            hi, lo = fn._ptrs(xs)
            _k(L.b2d_rf_start(noise.data_ptr(), 0 if gt_spec is None else gt_spec.data_ptr(), ts, one_m, spec_min,
                              spec_range, B, T, M, x.data_ptr(), hi, lo, _stream()), "b2d_rf_start")
            slot = lambda s: 0 if s is None else hist[s].data_ptr()
            draws = None if step_noise is None else iter(step_noise)
            for e, ev in enumerate(plan):
                G = fn._velocity(g, P, xs, srows[e], 0, crows, B, T)
                z = None
                if ev.noise:
                    z = torch.randn((B, 1, M, T), device=dev) if draws is None else next(draws).to(dev).contiguous()
                _k(L.b2d_df_update(G.data_ptr(), P["out_b"].data_ptr(), coefs[e].data_ptr(), x.data_ptr(), slot(ev.write),
                                   *(slot(s) for s in ev.reads), 0 if z is None else z.data_ptr(), B, T, M,
                                   x.data_ptr() if ev.store else 0, hi if ev.emit else 0, lo if ev.emit else 0, _stream()),
                   "b2d_df_update")
            out = torch.empty(B, T, M, dtype=torch.float32, device=dev)
            _k(L.b2d_rf_finish(x.data_ptr(), spec_min, spec_range, N * M, out.data_ptr(), _stream()), "b2d_rf_finish")
        return out
