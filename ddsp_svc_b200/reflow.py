"""The reflow model's sampler on the GPU: the velocity network NaiveV2Diff (reference reflow/naive_v2_diff.py:101-231) and
the rectified-flow ODE sampler RectifiedFlow (reflow/reflow.py), inference only.

Same constructors and parameter trees as the reference (a Unit2Wav checkpoint's ``reflow_model.velocity_fn.*`` keys load
strictly; the Conv1d weights keep their [O, K, 1] shapes), covering the configuration Unit2Wav builds
(reflow/vocoder.py:165): ``use_mlp=False``, ``conv_only=True``, no wavenet skip, no norm, ``conv_model_type='mode1'``,
kernel 31, expansion 2, ``dim`` a multiple of 64.  Any other option raises NotImplementedError in the constructor.

Execution: activations stay token-major [B, T, C]; the reference's [B, T, M] output is already token-major.  Once per
sampling call: every layer's condition projection as ONE GEMM [B T, M] x [M, n_layers dim], and the whole step schedule
(RK4's half steps included) through the sinusoidal embedding, its MLP and every layer's step projection, batched over all
evaluations.  Per velocity evaluation: the input-projection GEMM; per layer the pointwise GEMM (dim -> 4 dim),
unit2control.cu's GLU -> depthwise conv -> SiLU and the pointwise GEMM (2 dim -> dim); the output-projection GEMM.  The
stages between the GEMMs (GELU, residuals, conditioning, the ODE update, start and finish) are the kernels of
csrc/reflow.cu, which write the next GEMM's operand directly (fp32, or the TF32 halves in "3xtf32" mode).  The GEMMs run
at ``gemm_precision`` (unit2control._Gemm: "3xtf32" default, "fp32", "tf32").

Training (``infer=False``, the reflow loss) and any call under grad raise NotImplementedError.
"""
import math

import torch
import torch.nn as nn

from . import _lib
from .ops import _need_cuda_f32, _stream
from .unit2control import _ConvModule, _Gemm, _k, _split

_NO_TRAINING = ("%s: training (the reflow loss and its gradients) is not built; run inference with infer=True under "
                "torch.no_grad()")


class _DiffusionEmbedding(nn.Module):
    """parameter-free sinusoidal embedding (naive_v2_diff.py:15-29): index 0 of ``diffusion_embedding``"""

    def __init__(self, dim):
        super().__init__()
        self.dim = dim

    def forward(self, x):
        """x [E] diffusion steps -> [E, dim] fp32.  The frequencies are the reference's fp32 values (it builds them from
        an integer arange); argument, sin and cos are float64: the argument reaches 1000 rad, where an fp32 product alone
        is off by up to 3e-5 rad.  A few hundred values per sampling call."""
        half = self.dim // 2
        scale = math.log(10000) / (half - 1)
        freq = torch.exp(torch.arange(half, device=x.device) * -scale)
        arg = x.double()[:, None] * freq.double()[None, :]
        return torch.cat((arg.sin(), arg.cos()), dim=-1).float()


class _Layer(nn.Module):                          # naive_v2_diff.py:32-98 with conv_only, no wavenet skip
    def __init__(self, dim, dim_cond, expansion_factor, kernel_size):
        super().__init__()
        self.conformer = _ConvModule(dim, naive=True, expansion_factor=expansion_factor, kernel_size=kernel_size)
        self.norm = nn.LayerNorm(dim)            # in the reference's state dict, unused when conv_only
        self.diffusion_step_projection = nn.Conv1d(dim, dim, 1)
        self.condition_projection = nn.Conv1d(dim_cond, dim, 1)


def _under_grad(module, *inputs):
    return torch.is_grad_enabled() and (any(p.requires_grad for p in module.parameters()) or
                                        any(torch.is_tensor(t) and t.requires_grad for t in inputs))


class NaiveV2Diff(nn.Module):
    #: precision of the library GEMMs, see unit2control._Gemm: "3xtf32" (default), "fp32", "tf32"
    gemm_precision = "3xtf32"

    def __init__(self, mel_channels=128, dim=512, use_mlp=True, mlp_factor=4, condition_dim=256, num_layers=20,
                 expansion_factor=2, kernel_size=31, conv_only=True, wavenet_like=False, use_norm=False,
                 conv_model_type='mode1', conv_dropout=0.0, atten_dropout=0.1):
        super().__init__()
        unsupported = [name for name, bad in (("use_mlp=True", use_mlp), ("conv_only=False", not conv_only),
                                              ("wavenet_like=True", wavenet_like), ("use_norm=True", use_norm),
                                              ("conv_model_type=%r" % (conv_model_type,), conv_model_type != "mode1"),
                                              ("kernel_size=%r" % (kernel_size,), kernel_size != 31),
                                              ("expansion_factor=%r" % (expansion_factor,), expansion_factor != 2),
                                              ("dim=%r (not a multiple of 64)" % (dim,), dim <= 0 or dim % 64),
                                              ("conv_dropout=%r" % (conv_dropout,), conv_dropout != 0))
                       if bad]
        if unsupported:
            raise NotImplementedError("NaiveV2Diff: only the configuration Unit2Wav builds is implemented (use_mlp=False, "
                                      "conv_only=True, mode1, kernel 31, expansion 2, dim a multiple of 64, no dropout); "
                                      "got " + ", ".join(unsupported))
        self.wavenet_like = wavenet_like
        self.mask_cond_ratio = None
        self.input_projection = nn.Conv1d(mel_channels, dim, 1)
        self.diffusion_embedding = nn.Sequential(_DiffusionEmbedding(dim), nn.Linear(dim, dim * mlp_factor), nn.GELU(),
                                                 nn.Linear(dim * mlp_factor, dim))
        self.conditioner_projection = nn.Identity()
        self.residual_layers = nn.ModuleList([_Layer(dim, condition_dim, expansion_factor, kernel_size)
                                              for _ in range(num_layers)])
        self.output_projection = nn.Conv1d(dim, mel_channels, 1)
        nn.init.zeros_(self.output_projection.weight)
        self.dim, self.mel_channels, self.condition_dim = dim, mel_channels, condition_dim
        self.__dict__["_packed"] = None

    # ---- weights in the layouts the GEMMs want, rebuilt when a parameter changes (load_state_dict, .to) ----
    def _pack(self):
        key = (self.gemm_precision,) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        c = self.__dict__.get("_packed")
        if c is not None and c[0] == key:
            return c[1]
        w2 = lambda conv: conv.weight.detach()[:, :, 0].contiguous()
        layers = self.residual_layers
        P = dict(in_w=w2(self.input_projection), in_b=self.input_projection.bias.detach().contiguous(),
                 mlp1_w=self.diffusion_embedding[1].weight.detach(), mlp1_b=self.diffusion_embedding[1].bias.detach(),
                 mlp2_w=self.diffusion_embedding[3].weight.detach(), mlp2_b=self.diffusion_embedding[3].bias.detach(),
                 step_w=torch.cat([w2(Ly.diffusion_step_projection) for Ly in layers]),
                 step_b=torch.cat([Ly.diffusion_step_projection.bias.detach() for Ly in layers]),
                 cond_w=torch.cat([w2(Ly.condition_projection) for Ly in layers]),
                 cond_b=torch.cat([Ly.condition_projection.bias.detach() for Ly in layers]),
                 out_w=w2(self.output_projection), out_b=self.output_projection.bias.detach().contiguous())
        P["layers"] = []
        for Ly in layers:
            net = Ly.conformer.net
            P["layers"].append(dict(pw1_w=w2(net[2]), pw1_b=net[2].bias.detach(), dw_w=net[4].weight.detach()[:, 0, :].contiguous(),
                                    dw_b=net[4].bias.detach().contiguous(), pw2_w=w2(net[6]),
                                    pw2_b=net[6].bias.detach().contiguous()))
        if self.gemm_precision == "3xtf32":          # weights of every GEMM as TF32-exact (hi, lo) pairs, once per checkpoint
            for d in [P] + P["layers"]:
                for name in [n for n in d if n.endswith("_w") and n != "dw_w"]:
                    d[name] = _split(d[name].contiguous())
        self.__dict__["_packed"] = (key, P)
        return P

    # ---- building blocks ----
    def _step_rows(self, g, P, steps):
        """diffusion steps [E] -> every layer's step projection [E, n_layers dim] (embedding, MLP, projections)"""
        e = self.diffusion_embedding[0](steps)
        e = g.linear(e, P["mlp1_w"], P["mlp1_b"])
        e = g.linear(torch.nn.functional.gelu(e), P["mlp2_w"], P["mlp2_b"])
        return g.linear(e, P["step_w"], P["step_b"])

    def _cond_rows(self, g, P, cond_tm):
        """condition [B, T, M_cond] token-major -> every layer's condition projection [B T, n_layers dim] (one GEMM)"""
        return g.linear(cond_tm.reshape(-1, cond_tm.shape[-1]), P["cond_w"], P["cond_b"])

    @staticmethod
    def _operand(g, n, c, dev):
        """a [n, c] GEMM operand buffer: (hi, lo) in 3xtf32 mode, one fp32 tensor otherwise"""
        new = lambda: torch.empty(n, c, dtype=torch.float32, device=dev)
        return (new(), new()) if g.mode == "3xtf32" else new()

    @staticmethod
    def _ptrs(xs):
        return (xs[0].data_ptr(), xs[1].data_ptr()) if isinstance(xs, tuple) else (xs.data_ptr(), 0)

    def _velocity(self, g, P, xs, steps, step_stride, conds, B, T, out_bias=None):
        """one evaluation of the network: xs the input operand [B T, M] -> output projection [B T, M] (+ out_bias);
        steps: the step rows of this evaluation ([B or 1, n_layers dim] from row stride step_stride), conds [B T, n_layers dim]"""
        L, D, dev, N = _lib.lib(), self.dim, conds.device, B * T
        LD = D * len(P["layers"])
        G = g.mm(xs, P["in_w"])
        h = torch.empty(N, D, dtype=torch.float32, device=dev)
        us = self._operand(g, N, D, dev)
        uh, ul = self._ptrs(us)
        _k(L.b2d_rf_layer_input(G.data_ptr(), P["in_b"].data_ptr(), h.data_ptr(), 0, steps.data_ptr(), step_stride,
                                conds.data_ptr(), LD, B, T, D, uh, ul, _stream()), "b2d_rf_layer_input")
        inner = 2 * D
        s = torch.empty(N, inner, dtype=torch.float32, device=dev)
        for i, Ly in enumerate(P["layers"]):
            hh = g.mm(us, Ly["pw1_w"], Ly["pw1_b"])                                   # [B T, 4 dim]: value | gate
            _k(L.b2d_u2c_glu_dwconv_silu(hh.data_ptr(), Ly["dw_w"].data_ptr(), Ly["dw_b"].data_ptr(), s.data_ptr(), B, T, inner,
                                         Ly["dw_w"].shape[1], _stream()), "b2d_u2c_glu_dwconv_silu")
            G2 = g.mm(g.split(s), Ly["pw2_w"])
            last = i + 1 == len(P["layers"])
            sp = 0 if last else steps.data_ptr() + 4 * (i + 1) * D
            cp = 0 if last else conds.data_ptr() + 4 * (i + 1) * D
            _k(L.b2d_rf_layer_input(G2.data_ptr(), Ly["pw2_b"].data_ptr(), h.data_ptr(), 1, sp, step_stride, cp, LD, B, T, D,
                                    uh, ul, _stream()), "b2d_rf_layer_input")
        return g.mm(us, P["out_w"], out_bias)

    def forward(self, spec, diffusion_step, cond):
        """spec [B, 1, M, T] or [B, M, T], diffusion_step [B] (one step per utterance), cond [B, M_cond, T] -> the
        velocity in the layout of spec"""
        if _under_grad(self, spec, diffusion_step, cond):
            raise NotImplementedError(_NO_TRAINING % "NaiveV2Diff")
        four = spec.dim() == 4
        x = spec[:, 0] if four else spec
        if x.dim() != 3:
            raise ValueError("mel must be 3 dim tensor, but got %d" % x.dim())
        _need_cuda_f32("spec", x)
        _need_cuda_f32("cond", cond)
        B, M, T = x.shape
        if M != self.mel_channels or cond.shape != (B, self.condition_dim, T):
            raise ValueError("NaiveV2Diff: spec [B, %d, T] and cond [B, %d, T] expected, got %s and %s"
                             % (self.mel_channels, self.condition_dim, tuple(x.shape), tuple(cond.shape)))
        steps = torch.as_tensor(diffusion_step, device=x.device).reshape(-1).expand(B)
        x = x.contiguous()
        with torch.no_grad(), _Gemm(self.gemm_precision) as g:
            P = self._pack()
            srows = self._step_rows(g, P, steps).contiguous()                           # [B, n_layers dim]
            crows = self._cond_rows(g, P, cond.transpose(1, 2).contiguous())
            xs = self._operand(g, B * T, M, x.device)
            hi, lo = self._ptrs(xs)
            _k(_lib.lib().b2d_rf_start(x.data_ptr(), 0, 0.0, 1.0, 0.0, 1.0, B, T, M, 0, hi, lo, _stream()), "b2d_rf_start")
            v = self._velocity(g, P, xs, srows, srows.shape[1], crows, B, T, out_bias=P["out_b"])
            v = v.reshape(B, T, M).transpose(1, 2).contiguous()
        return v[:, None] if four else v


class RectifiedFlow(nn.Module):
    def __init__(self, velocity_fn, out_dims=128, spec_min=-12, spec_max=2):
        super().__init__()
        if not isinstance(velocity_fn, NaiveV2Diff):
            raise ValueError("RectifiedFlow: velocity_fn must be ddsp_svc_b200.NaiveV2Diff, got %s" % type(velocity_fn).__name__)
        self.velocity_fn = velocity_fn
        self.out_dims = out_dims
        self.spec_min = spec_min
        self.spec_max = spec_max

    def forward(self, condition, gt_spec=None, infer=True, infer_step=10, method='euler', t_start=0.0, use_tqdm=True):
        """condition [B, T, M] (the DDSP mel), gt_spec [B, T, M] or None -> the sampled mel [B, T, M] (reflow.py:59-105).
        The initial noise is ONE torch.randn((B, 1, M, T)) on condition's device, as in the reference, so seeded runs
        compare.  ``use_tqdm`` is accepted and ignored."""
        fn = self.velocity_fn
        if not infer or _under_grad(self, condition, gt_spec):
            raise NotImplementedError(_NO_TRAINING % "RectifiedFlow")
        _need_cuda_f32("condition", condition)
        B, T, Mc = condition.shape
        M, dev = self.out_dims, condition.device
        if M != fn.mel_channels or Mc != fn.condition_dim:
            raise ValueError("RectifiedFlow: out_dims / condition width do not match the velocity network")
        if t_start < 0.0:
            t_start = 0.0
        shape = (B, 1, M, T)
        if gt_spec is not None:
            _need_cuda_f32("gt_spec", gt_spec)
            if gt_spec.shape != (B, T, M):
                raise ValueError("RectifiedFlow: gt_spec must be [B, T, %d] like condition" % M)
        noise = torch.randn(shape, device=dev)
        return self._sample(condition, noise, gt_spec, infer_step, method, t_start)

    def _sample(self, condition, noise, gt_spec, infer_step, method, t_start):
        """forward after the noise draw: noise [B, 1, M, T] given"""
        fn, (B, T, _), M, dev = self.velocity_fn, condition.shape, self.out_dims, condition.device
        _need_cuda_f32("noise", noise)
        if noise.shape != (B, 1, M, T):
            raise ValueError("RectifiedFlow: noise must be [B, 1, %d, T]" % M)
        if gt_spec is None:
            # the reference writes torch.full((b,), 0): an int64 t whose first `t += dt` raises; t here is fp32 from 0
            t, gt, ts = torch.zeros(1), None, 0.0
            dt = 1.0 / infer_step
        else:
            t, gt, ts = torch.full((1,), float(t_start)), gt_spec.contiguous(), float(t_start)
            dt = (1.0 - ts) / infer_step
        if method not in ("euler", "rk4"):
            raise NotImplementedError(method)
        # the step schedule with the reference's fp32 arithmetic (t += dt, 1000 (t + 0.5 dt), ...); every utterance shares it
        sched = []
        for _ in range(infer_step):
            sched += [1000 * t] if method == "euler" else [1000 * t, 1000 * (t + 0.5 * dt), 1000 * (t + 0.5 * dt), 1000 * (t + dt)]
            t += dt
        noise = noise.contiguous()
        L, N = _lib.lib(), B * T
        with torch.no_grad(), _Gemm(fn.gemm_precision) as g:
            P = fn._pack()
            crows = fn._cond_rows(g, P, condition.contiguous())
            srows = fn._step_rows(g, P, torch.cat(sched).to(dev)).contiguous() if sched else None   # [E, n_layers dim]
            x = torch.empty(N, M, dtype=torch.float32, device=dev)
            acc = torch.empty_like(x) if method == "rk4" and sched else None
            xs = fn._operand(g, N, M, dev)
            hi, lo = fn._ptrs(xs)
            rng = float(self.spec_max - self.spec_min)
            _k(L.b2d_rf_start(noise.data_ptr(), 0 if gt is None else gt.data_ptr(), ts, 1.0 - ts, float(self.spec_min), rng,
                              B, T, M, x.data_ptr(), hi, lo, _stream()), "b2d_rf_start")
            stages = (-1,) if method == "euler" else (0, 1, 2, 3)
            for e in range(len(sched)):
                G = fn._velocity(g, P, xs, srows[e], 0, crows, B, T)
                _k(L.b2d_rf_ode_update(G.data_ptr(), P["out_b"].data_ptr(), x.data_ptr(), 0 if acc is None else acc.data_ptr(),
                                       stages[e % len(stages)], dt, N, M, hi, lo, _stream()), "b2d_rf_ode_update")
            out = torch.empty(B, T, M, dtype=torch.float32, device=dev)
            _k(L.b2d_rf_finish(x.data_ptr(), float(self.spec_min), rng, N * M, out.data_ptr(), _stream()), "b2d_rf_finish")
        return out
