"""Random-scale spectral loss of the DDSP training step on the GPU: drop-in for ddsp.loss.RSSLoss (reference
ddsp/loss.py:32-54, built by train.py:82 for configs/combsub.yaml and sins.yaml).

``RSSLoss(fft_min, fft_max, n_scale)(x_pred, x_true)`` draws its scales with the reference's own call
(``torch.randint(fft_min, fft_max, (n_scale,))`` on torch's CPU generator, so ``torch.manual_seed`` reproduces the
reference's scales) and evaluates every scale with the kernels of csrc/rss_loss.cu: Bluestein transforms for any
n_fft in [256, 2047], per-frame partial sums and a float64 finalize to a 0-dim CUDA loss, with no host
synchronisation once the per-size tables exist (the first use of a size builds its table with one host
synchronisation; ``RSSLoss.prebuild_tables()`` builds all of them up front).  When ``x_pred`` requires grad the loss is differentiable with respect to it: the backward kernel
recomputes both spectra from the inputs.

Not built (NotImplementedError): overlap != 0, scales outside [256, 2048], a gradient with respect to x_true.
"""
import ctypes

import torch

from . import _lib, bluestein
from .ops import _count, _need_cuda_f32, _stream

N_MIN, N_MAX = 256, 2047
MAX_SCALES = 64


def bluestein_size(n):
    """the transform size the kernels use for n_fft = n: the smallest of 1024 / 2048 / 4096 that is >= 2n - 1"""
    return bluestein.size(n, n)


def table_host(n):
    """float32 table of csrc/rss_loss.cu for n_fft = n (bluestein.py's layout, all n bins): [0] c = sqrt(sum w^2) as
    torchaudio computes it, the periodic Hann window (torch.hann_window), the chirp and FFT_M(chirp filter) / M"""
    n = int(n)
    L = _lib.lib().b2d_rss_table_floats(n)
    if L <= 0:
        raise ValueError("n_fft=%d outside [%d, %d]" % (n, N_MIN, N_MAX))
    window = torch.hann_window(n)
    t = bluestein.table_host(n, n, window.numpy(), head=[window.pow(2.0).sum().sqrt().item()])
    assert t.size == L
    return t


_cache = bluestein.TableCache(table_host)
_tables = _cache.tables


def table(n, device):
    """table_host(n) on ``device``, cached per (n, device)"""
    return _cache.get(n, device)


def prebuild_tables(device, fft_min=N_MIN, fft_max=N_MAX + 1):
    """Build the tables of every n_fft in [fft_min, fft_max) on ``device`` now.  A table is otherwise built on the first
    call that draws its size, with one host synchronisation; prebuilding moves all of them before training."""
    for n in range(int(fft_min), int(fft_max)):
        table(n, device)


def _checked(x_pred, x_true, n_ffts):
    _need_cuda_f32("x_pred", x_pred)
    if not isinstance(x_true, torch.Tensor) or not x_true.is_cuda:
        raise ValueError("x_true must be a CUDA tensor (the kernels have no CPU fallback)")
    if x_true.dtype == torch.float16:
        x_true = x_true.float()                         # exact: every float16 is a float32
    _need_cuda_f32("x_true", x_true)
    if x_pred.dim() != 2 or x_true.shape != x_pred.shape:
        raise ValueError("x_pred and x_true must both be [B, T], got %s and %s"
                         % (tuple(x_pred.shape), tuple(x_true.shape)))
    if x_true.device != x_pred.device:
        raise ValueError("x_true lives on %s, x_pred on %s" % (x_true.device, x_pred.device))
    n_ffts = [int(n) for n in n_ffts]
    if not 0 < len(n_ffts) <= MAX_SCALES:
        raise ValueError("1 to %d scales are supported, got %d" % (MAX_SCALES, len(n_ffts)))
    B, T = x_pred.shape
    for n in n_ffts:
        if not N_MIN <= n <= N_MAX:
            raise ValueError("n_fft=%d outside [%d, %d]" % (n, N_MIN, N_MAX))
        if T < n:
            raise ValueError("signal of %d samples is shorter than n_fft=%d" % (T, n))
    return x_pred.detach().contiguous(), x_true.detach().contiguous(), n_ffts


def _call_args(n_ffts, device):
    tabs = [table(n, device) for n in n_ffts]
    ns = (ctypes.c_int * len(n_ffts))(*n_ffts)
    ptrs = (ctypes.c_void_p * len(n_ffts))(*[t.data_ptr() for t in tabs])
    return ns, ptrs, tabs


def rss_loss_forward(x_pred, x_true, n_ffts, alpha=1.0, eps=1e-7):
    """-> (loss 0-dim fp32, norms [n_scale, B, 2] float64: ||S_t - S_p||, ||S_t + S_p|| per scale and row)"""
    x_pred, x_true, n_ffts = _checked(x_pred, x_true, n_ffts)
    B, T = x_pred.shape
    L = _lib.lib()
    ns, ptrs, _keep = _call_args(n_ffts, x_pred.device)
    ws_bytes = L.b2d_rss_loss_workspace_bytes(B, T, len(n_ffts), ns)
    ws = torch.empty(ws_bytes // 8, dtype=torch.float64, device=x_pred.device)
    norms = torch.empty(len(n_ffts), B, 2, dtype=torch.float64, device=x_pred.device)
    loss = torch.empty((), dtype=torch.float32, device=x_pred.device)
    _lib.check(L.b2d_rss_loss_forward(x_pred.data_ptr(), x_true.data_ptr(), B, T, len(n_ffts), ns, ptrs, float(alpha),
                                      float(eps), ws.data_ptr(), ws_bytes, norms.data_ptr(), loss.data_ptr(), _stream()),
               "b2d_rss_loss_forward")
    _count(len(n_ffts) + 1)
    return loss, norms


def rss_loss_backward(x_pred, x_true, n_ffts, norms, grad_loss, alpha=1.0, eps=1e-7):
    """dL/dx_pred [B, T] for dL/dloss ``grad_loss`` (0-dim CUDA tensor, read on the device) and the forward's norms.
    The spectra are recomputed from x_pred and x_true, so they must be the forward's inputs."""
    x_pred, x_true, n_ffts = _checked(x_pred, x_true, n_ffts)
    B, T = x_pred.shape
    _need_cuda_f32("grad_loss", grad_loss)
    grad_loss = grad_loss.reshape(()).contiguous()
    _need_cuda_f32("norms", norms, dtype=torch.float64)
    if tuple(norms.shape) != (len(n_ffts), B, 2):
        raise ValueError("norms must be [n_scale, B, 2], got %s" % (tuple(norms.shape),))
    norms = norms.contiguous()
    L = _lib.lib()
    ns, ptrs, _keep = _call_args(n_ffts, x_pred.device)
    grad = torch.empty(B, T, dtype=torch.float32, device=x_pred.device)
    _lib.check(L.b2d_rss_loss_backward(x_pred.data_ptr(), x_true.data_ptr(), B, T, len(n_ffts), ns, ptrs, float(alpha),
                                       float(eps), norms.data_ptr(), grad_loss.data_ptr(), grad.data_ptr(), _stream()),
               "b2d_rss_loss_backward")
    _count(len(n_ffts))
    return grad


class _RSSLossFn(torch.autograd.Function):
    """RSSLoss with a CUDA backward.  Saves the inputs, the scales and the per-(scale, row) norms only."""

    @staticmethod
    def forward(ctx, x_pred, x_true, n_ffts, alpha, eps):
        loss, norms = rss_loss_forward(x_pred, x_true, n_ffts, alpha, eps)
        ctx.n_ffts, ctx.alpha, ctx.eps = n_ffts, alpha, eps
        ctx.save_for_backward(x_pred, x_true, norms)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        x_pred, x_true, norms = ctx.saved_tensors
        grad = rss_loss_backward(x_pred, x_true, ctx.n_ffts, norms, grad_loss.float(), ctx.alpha, ctx.eps)
        return grad, None, None, None, None


class RSSLoss(torch.nn.Module):
    """Random-scale spectral loss (ddsp/loss.py:32-54): the reference's constructor and forward(x_pred, x_true).
    ``n_ffts=``: pin the scales of one call instead of drawing them.  Returns a 0-dim fp32 CUDA tensor."""

    def __init__(self, fft_min, fft_max, n_scale, alpha=1.0, overlap=0, eps=1e-7, device='cuda'):
        super().__init__()
        if overlap != 0:
            raise NotImplementedError("the RSS loss kernels use hop = n_fft (overlap=0, the reference's default); "
                                      "got overlap=%r" % (overlap,))
        if not (N_MIN <= fft_min < fft_max <= N_MAX + 1):
            raise NotImplementedError("the RSS loss kernels cover n_fft in [%d, %d] (fft_min >= %d, fft_max <= %d); "
                                      "got [%r, %r)" % (N_MIN, N_MAX, N_MIN, N_MAX + 1, fft_min, fft_max))
        if not 0 < int(n_scale) <= MAX_SCALES:
            raise NotImplementedError("n_scale must be in [1, %d], got %r" % (MAX_SCALES, n_scale))
        self.fft_min = fft_min
        self.fft_max = fft_max
        self.n_scale = n_scale
        self.alpha = float(alpha)
        self.eps = float(eps)
        self.device = device

    def prebuild_tables(self, device=None):
        """Build the per-size tables of every scale this loss can draw (see loss.prebuild_tables)."""
        prebuild_tables(self.device if device is None else device, self.fft_min, self.fft_max)

    def forward(self, x_pred, x_true, n_ffts=None):
        if isinstance(x_true, torch.Tensor) and x_true.requires_grad:
            raise NotImplementedError("RSSLoss has no gradient with respect to x_true (the training step needs the "
                                      "prediction's only); pass x_true.detach()")
        for name, x in (("x_pred", x_pred), ("x_true", x_true)):
            if not isinstance(x, torch.Tensor) or not x.is_cuda:
                raise ValueError("%s must be a CUDA tensor (the kernels have no CPU fallback)" % name)
        if n_ffts is None:
            n_ffts = torch.randint(self.fft_min, self.fft_max, (self.n_scale,))
        n_ffts = tuple(int(n) for n in (n_ffts.tolist() if isinstance(n_ffts, torch.Tensor) else n_ffts))
        if torch.is_grad_enabled() and x_pred.requires_grad:
            return _RSSLossFn.apply(x_pred, x_true, n_ffts, self.alpha, self.eps)
        return rss_loss_forward(x_pred, x_true, n_ffts, self.alpha, self.eps)[0]
