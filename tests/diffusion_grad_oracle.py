"""Plain-torch restatement of GaussianDiffusion's training loss (reference diffusion/diffusion.py:194-238: norm_spec,
q_sample, the denoiser, F.mse_loss with loss_type 'l2') around the oracle denoisers (tests/diffusion_oracle.WaveNet,
tests/reflow_oracle.VelocityNet), in the network's dtype (float64 for gradients against which the kernels are measured),
fed explicit draws.

TEST INFRASTRUCTURE ONLY.  tests/test_oracle_diffusion_grad.py pins it to the reference's own losses and float64
gradients stored by tests/golden/make_golden_diffusion_grad.py; the GPU tests use it where the reference does not exist.
"""
import torch
import torch.nn.functional as F

from tests import diffusion_oracle


def draws(B, T, t_max, M=128, device=None):
    """the reference's draws in its order (fp32 torch on `device`): t = torch.randint(0, t_max, (B,)), then the noise
    as randn_like of the transposed [B, 1, M, T] view, returned token-major [B, T, M]"""
    t = torch.randint(0, t_max, (B,), device=device).long()
    noise = torch.empty_strided((B, 1, M, T), (T * M, T * M, 1, M), device=device).normal_()
    return t, noise[:, 0].transpose(1, 2)


def oracle_loss(net, condition, gt, t, noise, spec_min=-12, spec_max=2):
    """condition [B, T, M_cond], gt [B, T, M], t [B] int64, noise [B, T, M] token-major -> loss [] in the network's
    dtype.  The schedule's coefficients are the registered fp32 buffers' values, as a float64 copy of the reference
    module would hold them."""
    dtype = net.input_projection.weight.dtype
    tb = diffusion_oracle.tables()
    a = tb["sqrt_alphas_cumprod"].to(gt.device, dtype)[t][:, None, None, None]
    b = tb["sqrt_one_minus_alphas_cumprod"].to(gt.device, dtype)[t][:, None, None, None]
    x0 = ((gt.to(dtype) - spec_min) / (spec_max - spec_min) * 2 - 1).transpose(1, 2)[:, None]
    n = noise.to(dtype).transpose(1, 2)[:, None]
    x_t = a * x0 + b * n
    return F.mse_loss(n, net(x_t, t, condition.to(dtype).transpose(1, 2)).reshape(n.shape))
