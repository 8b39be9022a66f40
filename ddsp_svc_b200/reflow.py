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

Training: with ``NaiveV2Diff.reflow_backward`` on, ``RectifiedFlow(infer=False)`` returns the reference's reflow loss
(loss_type 'l2_lognorm', the reference's draws of t and x_0) and NaiveV2Diff's forward under grad its velocity, both
differentiable with respect to the velocity network's parameters and the condition: ONE autograd Function each, whose
forward is the inference forward (same launches, bit-identical) plus the saved activations and whose backward walks the
layers in reverse on the kernels of csrc/reflow_bwd.cu and unit2control_bwd.cu and library GEMMs at ``gemm_precision``.
With the switch off (the default) infer=False and every call under grad raise NotImplementedError; with it on, the
sampler under grad still does.
"""
import math

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

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


def _network_backward(mod, g, S, gv, gvs, want_cond):
    """The velocity network's backward from gv [B T, M], the cotangent of its output (fp32), and gvs, that cotangent as
    the operand of the output projection's adjoints.  S: what _velocity / _step_rows / _cond_rows saved.  -> (dict of
    parameter gradients by name, the condition's cotangent [B T, M_cond] or None).

    Per layer, reversed: pw2's adjoints, the GLU-conv-SiLU backward recomputed from the saved pw1 output, pw1's adjoints,
    then rf_layer_backward adds g_z into the residual stream's cotangent and into column block i of G_Z.  Every layer's
    condition projection then takes ONE pair of GEMMs over G_Z [B T, n_layers dim], and the step projections the
    per-utterance token sums of G_Z; the step MLP's GEMMs have B rows."""
    P, (B, T) = S["P"], S["BT"]
    L, D, N, dev, nL = _lib.lib(), mod.dim, B * T, gv.device, len(S["P"]["layers"])
    LD, inner, split = nL * D, 2 * D, g.mode == "3xtf32"
    ws_bytes = L.b2d_u2c_backward_workspace_bytes(B, T, inner, max(mod.mel_channels, 4 * D, LD))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    rws_bytes = L.b2d_rf_backward_workspace_bytes(B, T, LD)
    rws = torch.empty(rws_bytes, dtype=torch.uint8, device=dev)
    new = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
    halves = lambda ops: mod._ptrs(ops) if split else (0, 0)       # fp32 modes: the fp32 tensor is the operand

    def colsum(x):
        out = new(x.shape[1])
        _k(L.b2d_u2c_colsum(x.data_ptr(), x.shape[0], x.shape[1], out.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
           "b2d_u2c_colsum")
        return out

    def gelu_backward(gy, pre, bias):
        """-> (fp32 cotangent of GELU's input, its operand)"""
        gx = new(*gy.shape)
        ops = mod._operand(g, gy.shape[0], gy.shape[1], dev) if split else gx
        hi, lo = halves(ops)
        _k(L.b2d_rf_gelu_backward(gy.data_ptr(), pre.data_ptr(), 0 if bias is None else bias.data_ptr(), gy.shape[0],
                                  gy.shape[1], gx.data_ptr(), hi, lo, _stream()), "b2d_rf_gelu_backward")
        return gx, ops

    G = {"output_projection.weight": g.grad_weight(gvs, S["hL"]).unsqueeze(-1), "output_projection.bias": colsum(gv)}
    gh = g.grad_input(gvs, P["out_w"])                                   # [B T, dim]: cotangent of h_L
    ghs = g.split(gh)
    gh_hi, gh_lo = halves(ghs)
    z = new(N, LD)                                                       # G_Z: every layer's g_z
    zs = mod._operand(g, N, LD, dev) if split else z
    z_hi, z_lo = halves(zs)
    for i in reversed(range(nL)):
        us, hh, ss = S["layers"][i]
        Ly, net = P["layers"][i], "residual_layers.%d.conformer.net." % i
        G[net + "6.weight"] = g.grad_weight(ghs, ss).unsqueeze(-1)
        G[net + "6.bias"] = colsum(gh)
        gs = g.grad_input(ghs, Ly["pw2_w"])                              # [B T, 2 dim]
        ghh, dwb = new(N, 2 * inner), new(inner, 32)
        _k(L.b2d_u2c_glu_dwconv_silu_backward(hh.data_ptr(), Ly["dw_w"].data_ptr(), Ly["dw_b"].data_ptr(), gs.data_ptr(),
                                              ghh.data_ptr(), dwb.data_ptr(), B, T, inner, Ly["dw_w"].shape[1], ws.data_ptr(),
                                              ws_bytes, _stream()), "b2d_u2c_glu_dwconv_silu_backward")
        G[net + "4.weight"], G[net + "4.bias"] = dwb[:, :31].unsqueeze(1).contiguous(), dwb[:, 31].contiguous()
        ghhs = g.split(ghh)
        G[net + "2.weight"] = g.grad_weight(ghhs, us).unsqueeze(-1)
        G[net + "2.bias"] = colsum(ghh)
        gz = g.grad_input(ghhs, Ly["pw1_w"])                             # [B T, dim]: cotangent of z_i
        _k(L.b2d_rf_layer_backward(gz.data_ptr(), gh.data_ptr(), B, T, D, i, nL, gh_hi, gh_lo, z.data_ptr(), z_hi, z_lo,
                                   rws.data_ptr(), rws_bytes, _stream()), "b2d_rf_layer_backward")
    # input projection: h_0 = GELU(in_proj(x_t)); x_t is data
    gpre, gpres = gelu_backward(gh, S["pre"], P["in_b"])
    G["input_projection.weight"] = g.grad_weight(gpres, S["xs"]).unsqueeze(-1)
    G["input_projection.bias"] = colsum(gpre)
    # every layer's condition projection at once
    dcw, dcb = g.grad_weight(zs, S["cond"]), colsum(z)
    g_cond = g.grad_input(zs, P["cond_w"]) if want_cond else None
    # step projections from the per-utterance sums of G_Z, then the step MLP (the sinusoidal embedding is data)
    gS = new(B, LD)
    _k(L.b2d_rf_step_sums(rws.data_ptr(), rws_bytes, B, T, LD, gS.data_ptr(), _stream()), "b2d_rf_step_sums")
    gSs = g.split(gS)
    dsw, dsb = g.grad_weight(gSs, g.split(S["e2"])), colsum(gS)
    ge2 = g.grad_input(gSs, P["step_w"])                                 # [B, dim]
    ge2s = g.split(ge2)
    G["diffusion_embedding.3.weight"] = g.grad_weight(ge2s, g.split(S["a1"]))
    G["diffusion_embedding.3.bias"] = colsum(ge2)
    ge1, ge1s = gelu_backward(g.grad_input(ge2s, P["mlp2_w"]), S["e1"], None)
    G["diffusion_embedding.1.weight"] = g.grad_weight(ge1s, g.split(S["e0"]))
    G["diffusion_embedding.1.bias"] = colsum(ge1)
    for i in range(nL):
        pre, rows = "residual_layers.%d." % i, slice(i * D, (i + 1) * D)
        G[pre + "condition_projection.weight"], G[pre + "condition_projection.bias"] = dcw[rows].unsqueeze(-1), dcb[rows]
        G[pre + "diffusion_step_projection.weight"] = dsw[rows].unsqueeze(-1)
        G[pre + "diffusion_step_projection.bias"] = dsb[rows]
    return G, g_cond


class _VelocityFunction(torch.autograd.Function):
    """NaiveV2Diff as ONE differentiable op: (module, parameter names, x [B, M, T], steps [B], cond [B, M_cond, T],
    *parameters) -> v [B T, M] token-major.  forward is NaiveV2Diff._run as it stands (same launches, same bits) plus
    the saved activations; backward is _network_backward.  x and steps are data.  Not differentiable twice."""

    @staticmethod
    def forward(ctx, mod, names, x, steps, cond, *params):
        S = {}
        with _Gemm(mod.gemm_precision) as g:
            v = mod._run(g, x, steps, cond, save=S)
        ctx.mod, ctx.names, ctx.saved, ctx.cond_shape = mod, names, S, cond.shape
        ctx.set_materialize_grads(False)
        return v

    @staticmethod
    @once_differentiable
    def backward(ctx, gv):
        if gv is None:
            return (None,) * (5 + len(ctx.names))
        mod, (B, Mc, T) = ctx.mod, ctx.cond_shape
        with _Gemm(mod.gemm_precision) as g:
            gv = gv.contiguous()
            G, g_cond = _network_backward(mod, g, ctx.saved, gv, g.split(gv), ctx.needs_input_grad[4])
        g_cond = None if g_cond is None else g_cond.reshape(B, T, Mc).transpose(1, 2)
        return (None, None, None, None, g_cond) + tuple(G.get(n) for n in ctx.names)


class _ReflowLossFunction(torch.autograd.Function):
    """The reflow loss with its velocity network as ONE differentiable op: (flow, parameter names, condition [B, T, M_cond],
    gt [B, T, M], t [B], x0 [B, T, M], w [B], *parameters) -> loss [].  forward is RectifiedFlow._loss_forward (rf_loss_input,
    the velocity network as NaiveV2Diff._velocity runs it, rf_loss); backward is rf_loss_backward, which writes the
    output projection's operand directly, then _network_backward.  gt, t, x0 and w are data.  Not differentiable twice."""

    @staticmethod
    def forward(ctx, flow, names, condition, gt, t, x0, w, *params):
        S = {}
        loss = flow._loss_forward(condition, gt, t, x0, w, save=S)
        ctx.flow, ctx.names, ctx.saved, ctx.w = flow, names, S, w
        ctx.set_materialize_grads(False)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, gl):
        if gl is None:
            return (None,) * (7 + len(ctx.names))
        mod, S = ctx.flow.velocity_fn, ctx.saved
        (B, T), M, dev = S["BT"], mod.mel_channels, gl.device
        gl = gl.reshape(1).to(torch.float32).contiguous()
        with _Gemm(mod.gemm_precision) as g:
            gv = torch.empty(B * T, M, dtype=torch.float32, device=dev)
            gvs = mod._operand(g, B * T, M, dev) if g.mode == "3xtf32" else gv
            hi, lo = mod._ptrs(gvs) if g.mode == "3xtf32" else (0, 0)
            _k(_lib.lib().b2d_rf_loss_backward(S["G"].data_ptr(), S["P"]["out_b"].data_ptr(), S["target"].data_ptr(),
                                               ctx.w.data_ptr(), gl.data_ptr(), B, T, M, gv.data_ptr(), hi, lo, _stream()),
               "b2d_rf_loss_backward")
            G, g_cond = _network_backward(mod, g, S, gv, gvs, ctx.needs_input_grad[2])
        g_cond = None if g_cond is None else g_cond.reshape(B, T, -1)
        return (None, None, g_cond, None, None, None, None) + tuple(G.get(n) for n in ctx.names)


class NaiveV2Diff(nn.Module):
    #: precision of the library GEMMs, see unit2control._Gemm: "3xtf32" (default), "fp32", "tf32"
    gemm_precision = "3xtf32"
    #: training: with grad mode on and a parameter (or cond) that requires grad, forward is differentiable with respect
    #: to the parameters and cond, and RectifiedFlow(infer=False) returns the reflow loss, differentiable with respect to
    #: the parameters and condition (the backward of _VelocityFunction / _ReflowLossFunction; the forward issues the same
    #: kernels with the same results).  Off by default: every call under grad and infer=False raise, and tests pin that.
    #: Set it on the class (``NaiveV2Diff.reflow_backward = True``) or per instance.
    reflow_backward = False

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
    def _step_rows(self, g, P, steps, save=None):
        """diffusion steps [E] -> every layer's step projection [E, n_layers dim] (embedding, MLP, projections);
        ``save``: a dict that receives the MLP's input, pre-activation and outputs"""
        e0 = self.diffusion_embedding[0](steps)
        e1 = g.linear(e0, P["mlp1_w"], P["mlp1_b"])
        a1 = torch.nn.functional.gelu(e1)
        e2 = g.linear(a1, P["mlp2_w"], P["mlp2_b"])
        if save is not None:
            save.update(e0=e0, e1=e1, a1=a1, e2=e2)
        return g.linear(e2, P["step_w"], P["step_b"])

    def _cond_rows(self, g, P, cond_tm, save=None):
        """condition [B, T, M_cond] token-major -> every layer's condition projection [B T, n_layers dim] (one GEMM);
        ``save``: a dict that receives the condition's operand"""
        cs = g.split(cond_tm.reshape(-1, cond_tm.shape[-1]))
        if save is not None:
            save["cond"] = cs
        return g.mm(cs, P["cond_w"], P["cond_b"])

    @staticmethod
    def _operand(g, n, c, dev):
        """a [n, c] GEMM operand buffer: (hi, lo) in 3xtf32 mode, one fp32 tensor otherwise"""
        new = lambda: torch.empty(n, c, dtype=torch.float32, device=dev)
        return (new(), new()) if g.mode == "3xtf32" else new()

    @staticmethod
    def _ptrs(xs):
        return (xs[0].data_ptr(), xs[1].data_ptr()) if isinstance(xs, tuple) else (xs.data_ptr(), 0)

    def _velocity(self, g, P, xs, steps, step_stride, conds, B, T, out_bias=None, save=None):
        """one evaluation of the network: xs the input operand [B T, M] -> output projection [B T, M] (+ out_bias);
        steps: the step rows of this evaluation ([B or 1, n_layers dim] from row stride step_stride), conds [B T, n_layers dim].
        ``save``: a dict that receives what the backward needs (then every layer gets its own buffers; same values)"""
        L, D, dev, N = _lib.lib(), self.dim, conds.device, B * T
        LD = D * len(P["layers"])
        G = g.mm(xs, P["in_w"])
        h = torch.empty(N, D, dtype=torch.float32, device=dev)
        us = self._operand(g, N, D, dev)
        uh, ul = self._ptrs(us)
        _k(L.b2d_rf_layer_input(G.data_ptr(), P["in_b"].data_ptr(), h.data_ptr(), 0, steps.data_ptr(), step_stride,
                                conds.data_ptr(), LD, B, T, D, uh, ul, _stream()), "b2d_rf_layer_input")
        if save is not None:
            save.update(xs=xs, pre=G, layers=[])
        inner = 2 * D
        s = torch.empty(N, inner, dtype=torch.float32, device=dev)
        for i, Ly in enumerate(P["layers"]):
            hh = g.mm(us, Ly["pw1_w"], Ly["pw1_b"])                                   # [B T, 4 dim]: value | gate
            if save is not None and i:
                s = torch.empty(N, inner, dtype=torch.float32, device=dev)
            _k(L.b2d_u2c_glu_dwconv_silu(hh.data_ptr(), Ly["dw_w"].data_ptr(), Ly["dw_b"].data_ptr(), s.data_ptr(), B, T, inner,
                                         Ly["dw_w"].shape[1], _stream()), "b2d_u2c_glu_dwconv_silu")
            ss = g.split(s)
            G2 = g.mm(ss, Ly["pw2_w"])
            if save is not None:                     # z_i operand, pw1 output, GLU-stage output operand
                save["layers"].append((us, hh, ss))
                us = self._operand(g, N, D, dev)
                uh, ul = self._ptrs(us)
            last = i + 1 == len(P["layers"])
            sp = 0 if last else steps.data_ptr() + 4 * (i + 1) * D
            cp = 0 if last else conds.data_ptr() + 4 * (i + 1) * D
            _k(L.b2d_rf_layer_input(G2.data_ptr(), Ly["pw2_b"].data_ptr(), h.data_ptr(), 1, sp, step_stride, cp, LD, B, T, D,
                                    uh, ul, _stream()), "b2d_rf_layer_input")
        if save is not None:
            save["hL"] = us
        return g.mm(us, P["out_w"], out_bias)

    def _run(self, g, x, steps, cond, save=None):
        """x [B, M, T] contiguous, steps [B], cond [B, M_cond, T] -> the velocity [B T, M] token-major (with the output
        bias); ``save``: a dict that receives what the backward needs"""
        B, M, T = x.shape
        P = self._pack()
        srows = self._step_rows(g, P, steps, save).contiguous()                          # [B, n_layers dim]
        crows = self._cond_rows(g, P, cond.transpose(1, 2).contiguous(), save)
        xs = self._operand(g, B * T, M, x.device)
        hi, lo = self._ptrs(xs)
        _k(_lib.lib().b2d_rf_start(x.data_ptr(), 0, 0.0, 1.0, 0.0, 1.0, B, T, M, 0, hi, lo, _stream()), "b2d_rf_start")
        if save is not None:
            save.update(P=P, BT=(B, T))
        return self._velocity(g, P, xs, srows, srows.shape[1], crows, B, T, out_bias=P["out_b"], save=save)

    def _grad_params(self):
        """(names, tensors) of the parameters the backward produces gradients for, in named_parameters order: all but the
        layers' LayerNorms (in the reference's state dict, never used when conv_only: their gradients stay None)"""
        items = [(n, p) for n, p in self.named_parameters() if not (n.startswith("residual_layers.") and ".norm." in n)]
        return tuple(n for n, _ in items), tuple(p for _, p in items)

    def forward(self, spec, diffusion_step, cond):
        """spec [B, 1, M, T] or [B, M, T], diffusion_step [B] (one step per utterance), cond [B, M_cond, T] -> the
        velocity in the layout of spec.  Under grad (``reflow_backward`` on): differentiable with respect to the
        parameters and cond, bit-identical to the no_grad call; spec and diffusion_step are data."""
        grad = _under_grad(self, spec, diffusion_step, cond)
        if grad and not self.reflow_backward:
            raise NotImplementedError(_NO_TRAINING % "NaiveV2Diff")
        if grad:
            for name, t in (("spec", spec), ("diffusion_step", diffusion_step)):
                if torch.is_tensor(t) and t.requires_grad:
                    raise NotImplementedError("NaiveV2Diff: no gradient with respect to %s (the reflow loss does not need "
                                              "it, so it is not built)" % name)
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
        if grad:
            names, params = self._grad_params()
            v = _VelocityFunction.apply(self, names, x, steps.detach(), cond, *params)
        else:
            with torch.no_grad(), _Gemm(self.gemm_precision) as g:
                v = self._run(g, x, steps, cond)
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
        compare.  ``use_tqdm`` is accepted and ignored.

        ``infer=False`` with ``NaiveV2Diff.reflow_backward`` on: the reference's reflow loss (reflow.py:20-35, :63-68,
        loss_type 'l2_lognorm') with its draws: t = t_start + (1 - t_start) torch.rand(B) clipped to [1e-7, 1 - 1e-7],
        then x_0 = torch.randn_like of the transposed [B, 1, M, T] view of norm(gt_spec), which is token-major in
        memory.  Differentiable with respect to the velocity network's parameters and condition; gt_spec is data."""
        fn = self.velocity_fn
        if not infer:
            if not fn.reflow_backward:
                raise NotImplementedError(_NO_TRAINING % "RectifiedFlow")
            return self._training_loss(condition, gt_spec, max(t_start, 0.0))
        if _under_grad(self, condition, gt_spec):
            raise NotImplementedError(_NO_TRAINING % "RectifiedFlow" if not fn.reflow_backward else
                                      "RectifiedFlow: the sampler (infer=True) is not differentiable; run it under "
                                      "torch.no_grad()")
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

    # ---- training ----
    def _training_loss(self, condition, gt_spec, t_start):
        """forward(infer=False): the reference's draws (fp32 torch, in its order), then _loss"""
        if gt_spec is None:
            raise ValueError("RectifiedFlow: infer=False needs gt_spec")
        B, T, M, dev = condition.shape[0], condition.shape[1], self.out_dims, condition.device
        t = t_start + (1.0 - t_start) * torch.rand(B, device=dev)
        t = torch.clip(t, 1e-7, 1 - 1e-7)
        # randn_like(x_1) of the transposed view keeps its strides (T M, T M, 1, M): the draw fills [B, T, M] in order
        x0 = torch.empty_strided((B, 1, M, T), (T * M, T * M, 1, M), device=dev).normal_()
        return self._loss(condition, gt_spec, t, x0[:, 0].transpose(1, 2))

    def _loss(self, condition, gt_spec, t, x0, loss_type="l2_lognorm"):
        """the reflow loss after the draws: condition [B, T, M_cond], gt_spec [B, T, M], t [B] (clipped), x0 [B, T, M]
        token-major -> loss [] fp32.  Under grad: differentiable with respect to the velocity network's parameters and
        condition; otherwise the same value without saving activations"""
        if loss_type != "l2_lognorm":
            raise NotImplementedError("RectifiedFlow: loss_type %r is not built (forward uses 'l2_lognorm')" % (loss_type,))
        fn, M = self.velocity_fn, self.out_dims
        for name, v in (("condition", condition), ("gt_spec", gt_spec), ("t", t), ("x0", x0)):
            _need_cuda_f32(name, v)
        B, T, Mc = condition.shape
        if M != fn.mel_channels or Mc != fn.condition_dim:
            raise ValueError("RectifiedFlow: out_dims / condition width do not match the velocity network")
        if gt_spec.shape != (B, T, M) or x0.shape != (B, T, M) or t.shape != (B,):
            raise ValueError("RectifiedFlow: gt_spec and x0 must be [B, T, %d] like condition, t [B]" % M)
        for name, v in (("gt_spec", gt_spec), ("t", t), ("x0", x0)):
            if v.requires_grad:
                raise NotImplementedError("RectifiedFlow: no gradient with respect to %s (data)" % name)
        w = 0.398942 / t / (1 - t) * torch.exp(-0.5 * torch.log(t / (1 - t)) ** 2)        # reflow.py:30
        args = (condition.contiguous(), gt_spec.contiguous(), t.contiguous(), x0.contiguous(), w.contiguous())
        if _under_grad(self, condition):
            names, params = fn._grad_params()
            return _ReflowLossFunction.apply(self, names, *args, *params)
        with torch.no_grad():
            return self._loss_forward(*args)

    def _loss_forward(self, condition, gt, t, x0, w, save=None):
        """the loss on the kernels: rf_loss_input, the velocity network, rf_loss.  ``save``: a dict that receives what the
        backward needs"""
        fn, (B, T, _), M, dev = self.velocity_fn, condition.shape, self.out_dims, condition.device
        L, N = _lib.lib(), B * T
        with _Gemm(fn.gemm_precision) as g:
            P = fn._pack()
            srows = fn._step_rows(g, P, 1000 * t, save).contiguous()                       # [B, n_layers dim]
            crows = fn._cond_rows(g, P, condition, save)
            xs = fn._operand(g, N, M, dev)
            hi, lo = fn._ptrs(xs)
            target = torch.empty(N, M, dtype=torch.float32, device=dev)
            _k(L.b2d_rf_loss_input(gt.data_ptr(), x0.data_ptr(), t.data_ptr(), float(self.spec_min),
                                   float(self.spec_max - self.spec_min), B, T, M, target.data_ptr(), hi, lo, _stream()),
               "b2d_rf_loss_input")
            G = fn._velocity(g, P, xs, srows, srows.shape[1], crows, B, T, save=save)
            ws_bytes = L.b2d_rf_backward_workspace_bytes(B, T, M)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            loss = torch.empty((), dtype=torch.float32, device=dev)
            _k(L.b2d_rf_loss(G.data_ptr(), P["out_b"].data_ptr(), target.data_ptr(), w.data_ptr(), B, T, M, ws.data_ptr(),
                             ws_bytes, loss.data_ptr(), _stream()), "b2d_rf_loss")
        if save is not None:
            save.update(P=P, BT=(B, T), G=G, target=target)
        return loss
