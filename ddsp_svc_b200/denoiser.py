"""What the two denoisers share: the diffusion models' WaveNet (diffusion.py) and the reflow model's NaiveV2Diff
(reflow.py), which GaussianDiffusion takes either of as ``denoise_fn``.

Both run token-major [B, T, C] from the same start (rf_start writes the input projection's operand), give their owners
the same three operations (``_step_rows``, ``_cond_rows``, ``_velocity``), keep their weights in a packed dict in the
layouts the GEMMs want and differentiate the same way: ONE autograd Function for the network (forward is the inference
forward plus the saved activations, backward the denoiser's ``_backward``) and ONE for a training loss around it (the
owner's ``_loss_forward``, then rf_loss_backward, then the denoiser's ``_backward``).  Here are that base class, the two
Functions and the pieces both backwards are made of; the layers themselves stay with each model.
"""
import math

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib
from .ops import _need_cuda_f32, _stream
from .unit2control import _Gemm, _k, _split

_NO_TRAINING = ("%s: training (the loss and the network's gradients) is off; turn it on with %s.%s = True, or run "
                "inference under torch.no_grad()")


class _DiffusionEmbedding(nn.Module):
    """parameter-free sinusoidal embedding (naive_v2_diff.py:15-29, wavenet.py:14-28)"""

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


def _under_grad(module, *inputs):
    return torch.is_grad_enabled() and (any(p.requires_grad for p in module.parameters()) or
                                        any(torch.is_tensor(t) and t.requires_grad for t in inputs))


class _NetworkFunction(torch.autograd.Function):
    """A denoiser as ONE differentiable op: (module, parameter names, x [B, M, T], steps [B], cond [B, M_cond, T],
    *parameters) -> its output [B T, M] token-major.  forward is the module's _run as it stands (same launches, same
    bits) plus the saved activations; backward is its _backward.  x and steps are data.  Not differentiable twice."""

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
            G, g_cond = mod._backward(g, ctx.saved, gv, g.split(gv), ctx.needs_input_grad[4])
        g_cond = None if g_cond is None else g_cond.reshape(B, T, Mc).transpose(1, 2)
        return (None, None, None, None, g_cond) + tuple(G.get(n) for n in ctx.names)


class _LossFunction(torch.autograd.Function):
    """A training loss around a denoiser as ONE differentiable op: (owner, denoiser, parameter names, condition
    [B, T, M_cond], data, *parameters) -> loss [].  forward is owner._loss_forward(condition, *data) (its input kernel,
    the denoiser as its _velocity runs it, rf_loss), which saves the loss's weights w and target with the activations;
    backward is rf_loss_backward, which writes the output projection's operand directly, then the denoiser's _backward.
    data (GaussianDiffusion: gt, t, noise; RectifiedFlow: gt, t, x0, w) is not differentiated.  Not differentiable
    twice."""

    @staticmethod
    def forward(ctx, owner, mod, names, condition, data, *params):
        S = {}
        loss = owner._loss_forward(condition, *data, save=S)
        ctx.mod, ctx.names, ctx.saved = mod, names, S
        ctx.set_materialize_grads(False)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, gl):
        if gl is None:
            return (None,) * (5 + len(ctx.names))
        mod, S = ctx.mod, ctx.saved
        (B, T), M, dev = S["BT"], mod.mel_channels, gl.device
        gl = gl.reshape(1).to(torch.float32).contiguous()
        with _Gemm(mod.gemm_precision) as g:
            gv = torch.empty(B * T, M, dtype=torch.float32, device=dev)
            gvs = mod._operand(g, B * T, M, dev) if g.mode == "3xtf32" else gv
            hi, lo = mod._ptrs(gvs) if g.mode == "3xtf32" else (0, 0)
            _k(_lib.lib().b2d_rf_loss_backward(S["G"].data_ptr(), S["P"]["out_b"].data_ptr(), S["target"].data_ptr(),
                                               S["w"].data_ptr(), gl.data_ptr(), B, T, M, gv.data_ptr(), hi, lo, _stream()),
               "b2d_rf_loss_backward")
            G, g_cond = mod._backward(g, S, gv, gvs, ctx.needs_input_grad[3])
        g_cond = None if g_cond is None else g_cond.reshape(B, T, -1)
        return (None, None, None, g_cond, None) + tuple(G.get(n) for n in ctx.names)


def _weighted_mse(G, out_b, target, w, B, T, M):
    """rf_loss: the mean over [B T, M] of w_b (target - (G + out_b))^2, G the output projection without its bias ->
    loss [] fp32"""
    L, dev = _lib.lib(), G.device
    ws_bytes = L.b2d_rf_backward_workspace_bytes(B, T, M)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    _k(L.b2d_rf_loss(G.data_ptr(), out_b.data_ptr(), target.data_ptr(), w.data_ptr(), B, T, M, ws.data_ptr(), ws_bytes,
                     loss.data_ptr(), _stream()), "b2d_rf_loss")
    return loss


class _Adjoint:
    """What a denoiser's backward works with: its GEMMs ``g``, the workspace of unit2control_bwd.cu's kernels and
    column sums (``inner`` channels, ``cols`` columns at most), the per-utterance slab sums of every layer's step-path
    cotangent (rf_layer_backward / df_layer_backward, ``step_cols`` columns) and the helpers below."""

    def __init__(self, mod, g, B, T, dev, inner, cols, step_cols):
        self.L, self.mod, self.g, self.B, self.T, self.dev = _lib.lib(), mod, g, B, T, dev
        self.split, self.step_cols = g.mode == "3xtf32", step_cols
        self.ws_bytes = self.L.b2d_u2c_backward_workspace_bytes(B, T, inner, cols)
        self.ws = torch.empty(self.ws_bytes, dtype=torch.uint8, device=dev)
        self.rws_bytes = self.L.b2d_rf_backward_workspace_bytes(B, T, step_cols)
        self.rws = torch.empty(self.rws_bytes, dtype=torch.uint8, device=dev)

    def new(self, *shape):
        return torch.empty(*shape, dtype=torch.float32, device=self.dev)

    def operand(self, n, c, fp32):
        """the [n, c] GEMM operand a kernel writes beside the fp32 tensor ``fp32``: fresh halves in 3xtf32 mode"""
        return self.mod._operand(self.g, n, c, self.dev) if self.split else fp32

    def halves(self, ops):
        return self.mod._ptrs(ops) if self.split else (0, 0)       # fp32 modes: the fp32 tensor is the operand

    def colsum(self, x):
        out = self.new(x.shape[1])
        _k(self.L.b2d_u2c_colsum(x.data_ptr(), x.shape[0], x.shape[1], out.data_ptr(), self.ws.data_ptr(), self.ws_bytes,
                                 _stream()), "b2d_u2c_colsum")
        return out


def _step_adjoint(A, S, P, G, act_backward, mlp):
    """The step path's backward, after every layer's: the step projections from the per-utterance sums of the layers'
    step cotangents (rf_step_sums), then the step MLP (the sinusoidal embedding is data).  act_backward(gy, pre) -> (the
    fp32 cotangent of the MLP activation's input, its operand); mlp: the names of the MLP's two Linear layers, whose
    gradients go into G.  -> the gradients of every layer's step projection, stacked: weight [step_cols, C], bias."""
    g = A.g
    gS = A.new(A.B, A.step_cols)
    _k(A.L.b2d_rf_step_sums(A.rws.data_ptr(), A.rws_bytes, A.B, A.T, A.step_cols, gS.data_ptr(), _stream()),
       "b2d_rf_step_sums")
    gSs = g.split(gS)
    dsw, dsb = g.grad_weight(gSs, g.split(S["e2"])), A.colsum(gS)
    ge2 = g.grad_input(gSs, P["step_w"])                                 # [B, C]
    ge2s = g.split(ge2)
    G[mlp[1] + ".weight"], G[mlp[1] + ".bias"] = g.grad_weight(ge2s, g.split(S["a1"])), A.colsum(ge2)
    ge1, ge1s = act_backward(g.grad_input(ge2s, P["mlp2_w"]), S["e1"])
    G[mlp[0] + ".weight"], G[mlp[0] + ".bias"] = g.grad_weight(ge1s, g.split(S["e0"])), A.colsum(ge1)
    return dsw, dsb


class _Denoiser(nn.Module):
    """Base of WaveNet and NaiveV2Diff.  A subclass builds the reference's module tree and supplies ``_name`` (for
    messages), ``_switch`` (the name of its public training switch), ``_out_4d``, ``_layout`` (the packed weights),
    ``_step_rows``, ``_cond_rows``, ``_velocity`` and ``_backward``; ``mel_channels``, ``condition_dim`` and ``dim``."""
    #: precision of the library GEMMs, see unit2control._Gemm: "3xtf32" (default), "fp32", "tf32"
    gemm_precision = "3xtf32"
    _name = _switch = None
    _out_4d = False               # True: forward returns [B, 1, M, T] always; False: the layout of spec

    def _trains(self):
        """the subclass's training switch (``WaveNet.diffusion_backward``, ``NaiveV2Diff.reflow_backward``)"""
        return getattr(self, self._switch)

    # ---- weights in the layouts the GEMMs want, rebuilt when a parameter changes (load_state_dict, .to) ----
    def _pack(self):
        key = (self.gemm_precision,) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        c = self.__dict__.get("_packed")
        if c is not None and c[0] == key:
            return c[1]
        P = self._layout()
        if self.gemm_precision == "3xtf32":          # weights of every GEMM as TF32-exact (hi, lo) pairs, once per checkpoint
            for d in [P] + P["layers"]:
                for name in [n for n in d if n.endswith("_w") and n != "dw_w"]:     # dw_w: the depthwise conv's taps
                    d[name] = _split(d[name])
        self.__dict__["_packed"] = (key, P)
        return P

    @staticmethod
    def _operand(g, n, c, dev):
        """a [n, c] GEMM operand buffer: (hi, lo) in 3xtf32 mode, one fp32 tensor otherwise"""
        new = lambda: torch.empty(n, c, dtype=torch.float32, device=dev)
        return (new(), new()) if g.mode == "3xtf32" else new()

    @staticmethod
    def _ptrs(xs):
        return (xs[0].data_ptr(), xs[1].data_ptr()) if isinstance(xs, tuple) else (xs.data_ptr(), 0)

    def _run(self, g, x, steps, cond, save=None):
        """x [B, M, T] contiguous, steps [B], cond [B, M_cond, T] -> the output [B T, M] token-major (with the output
        bias); ``save``: a dict that receives what the backward needs"""
        B, M, T = x.shape
        P = self._pack()
        srows = self._step_rows(g, P, steps, save).contiguous()                          # [B, n_layers C]
        crows = self._cond_rows(g, P, cond.transpose(1, 2).contiguous(), save)
        xs = self._operand(g, B * T, M, x.device)
        hi, lo = self._ptrs(xs)
        _k(_lib.lib().b2d_rf_start(x.data_ptr(), 0, 0.0, 1.0, 0.0, 1.0, B, T, M, 0, hi, lo, _stream()), "b2d_rf_start")
        if save is not None:
            save.update(P=P, BT=(B, T))
        return self._velocity(g, P, xs, srows, srows.shape[1], crows, B, T, out_bias=P["out_b"], save=save)

    def _has_grad(self, name):
        """whether the backward produces the gradient of parameter ``name``"""
        return True

    def _grad_params(self):
        """(names, tensors) of the parameters the backward produces gradients for, in named_parameters order"""
        items = [(n, p) for n, p in self.named_parameters() if self._has_grad(n)]
        return tuple(n for n, _ in items), tuple(p for _, p in items)

    def forward(self, spec, diffusion_step, cond):
        """spec [B, 1, M, T] or [B, M, T], diffusion_step [B] (or one value for every utterance), cond [B, M_cond, T]
        -> the output [B, 1, M, T], or [B, M, T] for a 3-dim spec unless ``_out_4d``.  Under grad (the training
        switch on): differentiable with respect to the parameters and cond, bit-identical to the no_grad call; spec
        and diffusion_step are data."""
        grad = _under_grad(self, spec, diffusion_step, cond)
        if grad and not self._trains():
            raise NotImplementedError(_NO_TRAINING % (self._name, self._name, self._switch))
        if grad:
            for name, t in (("spec", spec), ("diffusion_step", diffusion_step)):
                if torch.is_tensor(t) and t.requires_grad:
                    raise NotImplementedError("%s: no gradient with respect to %s (the training losses do not need it, "
                                              "so it is not built)" % (self._name, name))
        four = spec.dim() == 4
        x = spec[:, 0] if four else spec
        if x.dim() != 3:
            raise ValueError("mel must be 3 dim tensor, but got %d" % x.dim())
        _need_cuda_f32("spec", x)
        _need_cuda_f32("cond", cond)
        B, M, T = x.shape
        if M != self.mel_channels or cond.shape != (B, self.condition_dim, T):
            raise ValueError("%s: spec [B, 1, %d, T] or [B, %d, T] and cond [B, %d, T] expected, got %s and %s"
                             % (self._name, self.mel_channels, self.mel_channels, self.condition_dim, tuple(spec.shape),
                                tuple(cond.shape)))
        steps = torch.as_tensor(diffusion_step, device=x.device).reshape(-1).expand(B)
        x = x.contiguous()
        if grad:
            names, params = self._grad_params()
            v = _NetworkFunction.apply(self, names, x, steps.detach(), cond, *params)
        else:
            with torch.no_grad(), _Gemm(self.gemm_precision) as g:
                v = self._run(g, x, steps, cond)
        v = v.reshape(B, T, M).transpose(1, 2).contiguous()
        return v[:, None] if four or self._out_4d else v
