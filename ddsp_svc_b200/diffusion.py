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

Training: with the denoiser's switch on (``WaveNet.diffusion_backward``; for NaiveV2Diff its own
``reflow_backward``), ``GaussianDiffusion(infer=False)`` returns the reference's loss (p_losses, loss_type 'l2', with
the reference's draws of t and the noise) and WaveNet's forward under grad its prediction, both differentiable with
respect to the denoiser's parameters and the condition: ONE autograd Function each, shared with NaiveV2Diff
(denoiser.py), whose forward is the inference forward (same launches, bit-identical) plus the saved activations and
whose backward, the denoiser's _backward, walks the layers in reverse -- WaveNet's on the kernels of csrc/diffusion_bwd.cu
(and reflow_bwd.cu's loss and step sums) and library GEMMs at ``gemm_precision``.  With the switch off (the default)
infer=False and every call under grad raise NotImplementedError; with it on, the samplers under grad still do.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from .denoiser import _Adjoint, _DiffusionEmbedding, _Denoiser, _LossFunction, _step_adjoint, _under_grad, _weighted_mse
from .ops import _need_cuda_f32, _stream
from .reflow import NaiveV2Diff
from .unit2control import _Gemm, _k

_NO_TRAINING = ("%s: training (p_losses and the denoiser's gradients) is off; turn it on with WaveNet.diffusion_backward "
                "= True (NaiveV2Diff.reflow_backward = True for that denoiser), or run inference with infer=True under "
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


class WaveNet(_Denoiser):
    #: training: with grad mode on and a parameter (or cond) that requires grad, forward is differentiable with respect
    #: to the parameters and cond, and GaussianDiffusion(infer=False) around this network returns the diffusion loss,
    #: differentiable with respect to the parameters and condition (the backward of denoiser._NetworkFunction /
    #: _LossFunction; the forward issues the same kernels with the same results).  Off by default: every call under
    #: grad and infer=False raise.  Set it on the class (``WaveNet.diffusion_backward = True``) or per instance.
    diffusion_backward = False
    _name, _switch, _out_4d = "WaveNet", "diffusion_backward", True

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

    def _layout(self):
        """the weights in the layouts the GEMMs want (_Denoiser._pack caches them)"""
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
        return P

    # ---- the sampler's three operations (the same names and signatures as NaiveV2Diff's) ----
    def _step_rows(self, g, P, steps, save=None):
        """diffusion steps [E] -> every layer's step projection [E, n_layers C] (embedding, MLP, projections);
        ``save``: a dict that receives the MLP's input, pre-activation and outputs"""
        e0 = self.diffusion_embedding(steps)
        e1 = g.linear(e0, P["mlp1_w"], P["mlp1_b"])
        a1 = F.mish(e1)
        e2 = g.linear(a1, P["mlp2_w"], P["mlp2_b"])
        if save is not None:
            save.update(e0=e0, e1=e1, a1=a1, e2=e2)
        return g.linear(e2, P["step_w"], P["step_b"])

    def _cond_rows(self, g, P, cond_tm, save=None):
        """condition [B, T, n_hidden] token-major -> every layer's condition projection plus both biases
        [B T, n_layers 2 C] (one GEMM); ``save``: a dict that receives the condition's operand and the rows"""
        cs = g.split(cond_tm.reshape(-1, cond_tm.shape[-1]))
        rows = g.mm(cs, P["cond_w"], P["cond_b"])
        if save is not None:
            save.update(cond=cs, crows=rows)
        return rows

    def _velocity(self, g, P, xs, steps, step_stride, conds, B, T, out_bias=None, save=None):
        """one evaluation of the denoiser: xs the input operand [B T, M] -> output projection [B T, M] (+ out_bias);
        steps: the step rows of this evaluation ([B or 1, n_layers C] from row stride step_stride), conds
        [B T, n_layers 2 C].  ``save``: a dict that receives what the backward needs (then every operand gets its own
        buffer; same launches, same values)"""
        L, C, dev, N, nL = _lib.lib(), self.dim, conds.device, B * T, len(P["layers"])
        new = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        h, skip = new(N, C), new(N, C)
        us, vs = self._operand(g, N, 3 * C, dev), self._operand(g, N, C, dev)
        (uh, ul), (vh, vl) = self._ptrs(us), self._ptrs(vs)
        G = g.mm(xs, P["in_w"])
        _k(L.b2d_df_layer(G.data_ptr(), P["in_b"].data_ptr(), h.data_ptr(), 0, 0, steps.data_ptr(), step_stride, 1.0, B, T,
                          C, uh, ul, _stream()), "b2d_df_layer")
        if save is not None:
            save.update(xs=xs, pre=G, layers=[])
        skip_div = math.sqrt(nL)
        for i, Ly in enumerate(P["layers"]):
            Z = g.mm(us, Ly["conv_w"])                                                   # [B T, 2 C]
            _k(L.b2d_df_gate(Z.data_ptr(), conds.data_ptr() + 4 * i * 2 * C, conds.shape[1], N, C, vh, vl, _stream()),
               "b2d_df_gate")
            R = g.mm(vs, Ly["out_w"])                                                    # [B T, 2 C]: residual | skip
            last = i + 1 == nL
            if save is not None:                     # the convolution operand, its product, the gate's operand
                save["layers"].append((us, Z, vs))
                if not last:
                    us = self._operand(g, N, 3 * C, dev)
                vs = self._operand(g, N, C, dev)
                (uh, ul), (vh, vl) = self._ptrs(us), self._ptrs(vs)
            sp = 0 if last else steps.data_ptr() + 4 * (i + 1) * C
            oh, ol = (vh, vl) if last else (uh, ul)
            _k(L.b2d_df_layer(R.data_ptr(), Ly["out_b"].data_ptr(), h.data_ptr(), skip.data_ptr(), 1 if i == 0 else 2, sp,
                              step_stride, skip_div, B, T, C, oh, ol, _stream()), "b2d_df_layer")
        S = g.mm(vs, P["skip_w"])
        if save is not None:                         # the skip projection's operand and product
            save.update(sk=vs, S=S)
            vs = self._operand(g, N, C, dev)
            vh, vl = self._ptrs(vs)
        _k(L.b2d_df_relu(S.data_ptr(), P["skip_b"].data_ptr(), N, C, vh, vl, _stream()), "b2d_df_relu")
        if save is not None:
            save["q"] = vs
        return g.mm(vs, P["out_w"], out_bias)

    def _backward(self, g, S, gv, gvs, want_cond):
        """WaveNet's backward from gv [B T, M], the cotangent of its output (fp32), and gvs, that cotangent as the
        operand of the output projection's adjoints.  S: what _velocity / _step_rows / _cond_rows saved.  -> (dict of
        parameter gradients by name, the condition's cotangent [B T, n_hidden] or None).

        Output side: the output projection's adjoints, df_relu_backward at the skip projection, its adjoints; every
        layer's skip output receives the same cotangent (g_p W_skip) / sqrt(n_layers).  Per layer, reversed: g_R =
        [g_h' / sqrt 2 | g_skip] (df_layer_backward writes it), the output projection's adjoints, df_gate_backward into
        column block i of G_Z, the convolution's adjoints over the saved [B T, 3 C] operand, then df_layer_backward
        (the adjoint of the operand's scatter, g_h, the next g_R, the step sums).  Every layer's condition projection
        then takes ONE pair of GEMMs over G_Z [B T, n_layers 2 C], whose column sums are both the condition
        projection's and the convolution's bias gradients; the step projections take the per-utterance token sums of
        g_y; the step MLP's GEMMs have B rows."""
        P, (B, T) = S["P"], S["BT"]
        C, N, nL = self.dim, B * T, len(P["layers"])
        LC, Z2 = nL * C, nL * 2 * C
        A = _Adjoint(self, g, B, T, gv.device, 2 * C, max(self.mel_channels, 4 * C, Z2), LC)
        L, new, operand, halves, colsum = A.L, A.new, A.operand, A.halves, A.colsum
        cols = lambda ops, blk: tuple(o[:, blk] for o in ops) if A.split else ops[:, blk]

        def relu_backward(gy, pre, bias):
            """-> (fp32 cotangent of ReLU(pre + bias)'s input, its operand)"""
            gx = new(*gy.shape)
            ops = operand(gy.shape[0], gy.shape[1], gx)
            hi, lo = halves(ops)
            _k(L.b2d_df_relu_backward(gy.data_ptr(), pre.data_ptr(), bias.data_ptr(), gy.shape[0], gy.shape[1],
                                      gx.data_ptr(), hi, lo, _stream()), "b2d_df_relu_backward")
            return gx, ops

        def mish_backward(gy, pre):
            """-> (fp32 cotangent of Mish(pre)'s input, its operand)"""
            gx = new(*gy.shape)
            _k(L.b2d_df_mish_backward(gy.data_ptr(), pre.data_ptr(), gy.numel(), gx.data_ptr(), 0, 0, _stream()),
               "b2d_df_mish_backward")
            return gx, g.split(gx)

        w3 = lambda x: x.unsqueeze(-1)
        G = {"output_projection.weight": w3(g.grad_weight(gvs, S["q"])), "output_projection.bias": colsum(gv)}
        gp, gps = relu_backward(g.grad_input(gvs, P["out_w"]), S["S"], P["skip_b"])
        G["skip_projection.weight"], G["skip_projection.bias"] = w3(g.grad_weight(gps, S["sk"])), colsum(gp)
        gsk = g.grad_input(gps, P["skip_w"])                             # [B T, C]; / sqrt(n_layers) in df_layer_backward
        skip_div = math.sqrt(nL)
        gh = new(N, C)
        gr = new(N, 2 * C)
        grs = operand(N, 2 * C, gr)
        gr_hi, gr_lo = halves(grs)
        _k(L.b2d_df_layer_backward(0, gh.data_ptr(), gsk.data_ptr(), skip_div, B, T, C, nL - 1, nL, gr.data_ptr(), gr_hi,
                                   gr_lo, 0, 0, _stream()), "b2d_df_layer_backward")    # h_L feeds nothing: g_R = [0 | g_skip]
        z = new(N, Z2)                                                   # G_Z: every layer's g_z
        zs = operand(N, Z2, z)
        z_hi, z_lo = halves(zs)
        crows = S["crows"]
        for i in reversed(range(nL)):
            us, Zi, vs = S["layers"][i]
            Ly, pre = P["layers"][i], "residual_layers.%d." % i
            G[pre + "output_projection.weight"] = w3(g.grad_weight(grs, vs))
            G[pre + "output_projection.bias"] = colsum(gr)
            ga = g.grad_input(grs, Ly["out_w"])                          # [B T, C]: cotangent of the gate's output
            _k(L.b2d_df_gate_backward(ga.data_ptr(), Zi.data_ptr(), crows.data_ptr() + 4 * i * 2 * C, Z2, N, C, i, nL,
                                      z.data_ptr(), z_hi, z_lo, _stream()), "b2d_df_gate_backward")
            gzs = cols(zs, slice(i * 2 * C, (i + 1) * 2 * C))
            dW = g.grad_weight(gzs, us)                                  # [2 C, 3 C]: column block k is tap k
            G[pre + "dilated_conv.weight"] = dW.reshape(2 * C, 3, C).permute(0, 2, 1).contiguous()
            gu = g.grad_input(gzs, Ly["conv_w"])                         # [B T, 3 C]
            nxt = i > 0
            _k(L.b2d_df_layer_backward(gu.data_ptr(), gh.data_ptr(), gsk.data_ptr(), skip_div, B, T, C, i, nL,
                                       gr.data_ptr() if nxt else 0, gr_hi if nxt else 0, gr_lo if nxt else 0,
                                       A.rws.data_ptr(), A.rws_bytes, _stream()), "b2d_df_layer_backward")
        # input projection: h_0 = ReLU(in_proj(x_t)); x_t is data
        gpre, gpres = relu_backward(gh, S["pre"], P["in_b"])
        G["input_projection.weight"], G["input_projection.bias"] = w3(g.grad_weight(gpres, S["xs"])), colsum(gpre)
        # every layer's condition projection at once; its bias and the convolution's share G_Z's column sums
        dcw, dcb = g.grad_weight(zs, S["cond"]), colsum(z)
        g_cond = g.grad_input(zs, P["cond_w"]) if want_cond else None
        # step projections from the per-utterance sums of g_y, then the step MLP
        dsw, dsb = _step_adjoint(A, S, P, G, mish_backward, ("mlp.0", "mlp.2"))
        for i in range(nL):
            pre, zr, sr = "residual_layers.%d." % i, slice(i * 2 * C, (i + 1) * 2 * C), slice(i * C, (i + 1) * C)
            G[pre + "conditioner_projection.weight"] = w3(dcw[zr])
            G[pre + "conditioner_projection.bias"] = dcb[zr]
            G[pre + "dilated_conv.bias"] = dcb[zr].clone()
            G[pre + "diffusion_projection.weight"], G[pre + "diffusion_projection.bias"] = dsw[sr], dsb[sr]
        return G, g_cond


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
        seeded runs compare.  ``use_tqdm`` is accepted and ignored.

        ``infer=False`` with the denoiser's switch on (``WaveNet.diffusion_backward``, ``NaiveV2Diff.reflow_backward``):
        the reference's training loss (diffusion.py:194-238, loss_type 'l2') with its draws: t = torch.randint(0, t_max,
        (B,)) with t_max = k_step, or self.k_step when k_step is None, then the noise as randn_like of the transposed
        [B, 1, M, T] view of norm(gt_spec), which is token-major in memory.  Differentiable with respect to the
        denoiser's parameters and condition; gt_spec is data."""
        training = self.denoise_fn._trains()
        if not infer:
            if not training:
                raise NotImplementedError(_NO_TRAINING % "GaussianDiffusion")
            return self._training_loss(condition, gt_spec, k_step)
        if _under_grad(self, condition, gt_spec):
            raise NotImplementedError(_NO_TRAINING % "GaussianDiffusion" if not training else
                                      "GaussianDiffusion: the samplers (infer=True) are not differentiable; run them "
                                      "under torch.no_grad()")
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

    # ---- training ----
    def _training_loss(self, condition, gt_spec, k_step):
        """forward(infer=False): the reference's draws (torch, on condition's device, in its order), then _loss"""
        if gt_spec is None:
            raise ValueError("GaussianDiffusion: infer=False needs gt_spec")
        B, T, M, dev = condition.shape[0], condition.shape[1], self.out_dims, condition.device
        t_max = self.k_step if k_step is None else k_step
        if not 0 < t_max <= self.num_timesteps:
            raise ValueError("GaussianDiffusion: k_step must be in [1, %d] (the schedule's length), got %r"
                             % (self.num_timesteps, t_max))
        t = torch.randint(0, t_max, (B,), device=dev).long()
        # randn_like(x_start) of the transposed view keeps its strides (T M, T M, 1, M): the draw fills [B, T, M] in order
        noise = torch.empty_strided((B, 1, M, T), (T * M, T * M, 1, M), device=dev).normal_()
        return self._loss(condition, gt_spec, t, noise[:, 0].transpose(1, 2))

    def _loss(self, condition, gt_spec, t, noise):
        """the diffusion loss after the draws: condition [B, T, M_cond], gt_spec [B, T, M], t [B] int64 (steps in
        [0, num_timesteps)), noise [B, T, M] token-major -> loss [] fp32, F.mse_loss(noise, denoise_fn(q_sample(...))).
        Under grad: differentiable with respect to the denoiser's parameters and condition; otherwise the same value
        without saving activations"""
        fn, M = self.denoise_fn, self.out_dims
        if not fn._trains():
            raise NotImplementedError(_NO_TRAINING % "GaussianDiffusion")
        for name, v in (("condition", condition), ("gt_spec", gt_spec), ("noise", noise)):
            _need_cuda_f32(name, v)
        B, T, Mc = condition.shape
        if M != fn.mel_channels or Mc != fn.condition_dim:
            raise ValueError("GaussianDiffusion: out_dims / condition width do not match the denoiser")
        if gt_spec.shape != (B, T, M) or noise.shape != (B, T, M) or t.shape != (B,):
            raise ValueError("GaussianDiffusion: gt_spec and noise must be [B, T, %d] like condition, t [B]" % M)
        if t.dtype != torch.int64 or t.device != condition.device:
            raise ValueError("GaussianDiffusion: t must be an int64 tensor on condition's device")
        for name, v in (("gt_spec", gt_spec), ("noise", noise)):
            if v.requires_grad:
                raise NotImplementedError("GaussianDiffusion: no gradient with respect to %s (data)" % name)
        args = (condition.contiguous(), gt_spec.contiguous(), t.contiguous(), noise.contiguous())
        if _under_grad(self, condition):
            names, params = fn._grad_params()
            return _LossFunction.apply(self, fn, names, args[0], args[1:], *params)
        with torch.no_grad():
            return self._loss_forward(*args)

    def _loss_forward(self, condition, gt, t, noise, save=None):
        """the loss on the kernels: df_loss_input (q_sample with the steps gathered on the device), the denoiser,
        rf_loss with w = 1 and target = noise (its mean of (target - v)^2 is F.mse_loss).  ``save``: a dict that
        receives what the backward needs"""
        fn, (B, T, _), M, dev = self.denoise_fn, condition.shape, self.out_dims, condition.device
        L, N = _lib.lib(), B * T
        buf = self._host()
        spec_min, spec_range = float(buf["spec_min"][0]), float(buf["spec_max"][0] - buf["spec_min"][0])
        with _Gemm(fn.gemm_precision) as g:
            P = fn._pack()
            srows = fn._step_rows(g, P, t, save).contiguous()                              # [B, n_layers C]
            crows = fn._cond_rows(g, P, condition, save)
            xs = fn._operand(g, N, M, dev)
            hi, lo = fn._ptrs(xs)
            sa, s1m = self.sqrt_alphas_cumprod.contiguous(), self.sqrt_one_minus_alphas_cumprod.contiguous()
            _k(L.b2d_df_loss_input(gt.data_ptr(), noise.data_ptr(), t.data_ptr(), sa.data_ptr(), s1m.data_ptr(), sa.numel(),
                                   spec_min, spec_range, B, T, M, hi, lo, _stream()),
               "b2d_df_loss_input")
            G = fn._velocity(g, P, xs, srows, srows.shape[1], crows, B, T, save=save)
            w = torch.ones(B, dtype=torch.float32, device=dev)
            loss = _weighted_mse(G, P["out_b"], noise, w, B, T, M)
        if save is not None:
            save.update(P=P, BT=(B, T), G=G, target=noise, w=w)
        return loss
