"""Training loss of the diffusion models on the kernels: GaussianDiffusion(infer=False) forward and forward + backward
around the configurations' denoisers, each alternated with the same loss around the denoiser written in plain torch
(tests/diffusion_oracle.py, tests/reflow_oracle.py) run eagerly in fp32 under torch's defaults -- cuDNN convolutions in
TF32, what the reference runs today.  Prints one JSON line, with the card's name and power limit read in the same run.
Writes nothing.

    python bench_diffusion_grad.py [--steps K] [--warmup W]

Rows: diffusion-new.yaml's WaveNet(128, 20, 512, 256) at 36 x 2 s (172 frames) and 32 x 10 s (861 frames);
diffusion.yaml's (the same network, t_max 300) and diffusion-fast.yaml's NaiveV2Diff(512, 6 layers, condition 128) at
48 x 172.  Step rows: the whole diffusion-new.yaml training step at 36 x 172 and 32 x 861 (Unit2Wav, diffusion/vocoder.py:
CombSubFast with its PCmer control network, infer=False -> get_mel -> mse, plus the diffusion loss on the control
network's hidden output -> backward through all of it); its eager arm runs the control network as the plain-torch
tests/u2c_pcmer_oracle.py network and the WaveNet as tests/diffusion_oracle.py (CombSubFast and get_mel are the package's
in both arms).  Every call is timed with CUDA events after the L2 was flushed (256 MiB memset, untimed); the arms alternate
call by call; medians of K calls after W warm-up calls of each.  Also reported: the GEMM FLOP of one loss forward and
backward from shapes, and the memory the training forward holds for its backward (allocated after a forward under grad,
minus the same after the no_grad forward), for both arms.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_reflow_grad import alternate, card, held  # noqa: E402

M = 128
ROWS = [("diffusion_new_yaml_b36_2s", "wavenet", 36, 172, 100), ("diffusion_new_yaml_b32_10s", "wavenet", 32, 861, 100),
        ("diffusion_yaml_b48_2s", "wavenet", 48, 172, 300), ("diffusion_fast_yaml_b48_2s", "naive", 48, 172, 100)]


STEP_ROWS = [("diffusion_new_yaml_step_b36_2s", 36, 172), ("diffusion_new_yaml_step_b32_10s", 32, 861)]


def gemm_flop(kind, B, T):
    """multiply-adds x 2 of the loss's GEMMs from shapes (the B-row step MLP is negligible): forward, and backward (two
    products per forward product, one for the input projection: none towards the noisy mel)"""
    N = B * T
    if kind == "wavenet":
        C, L, H = 512, 20, 256
        per_layer = 2 * C * 3 * C + C * 2 * C                        # the k = 3 convolution, the output projection
        fwd = 2 * N * (M * C + L * per_layer + L * H * 2 * C + C * C + C * M)
        bwd = 2 * N * (M * C + 2 * (L * per_layer + L * H * 2 * C + C * C + C * M))
    else:
        D, L, H = 512, 6, 128
        per_layer = D * 4 * D + 2 * D * D
        fwd = 2 * N * (M * D + L * per_layer + H * L * D + D * M)
        bwd = 2 * N * (M * D + 2 * (L * per_layer + H * L * D + D * M))
    return fwd, bwd


def run_row(kind, B, T, t_max, flush, steps, warmup):
    import torch
    import ddsp_svc_b200 as pkg
    from tests import diffusion_grad_oracle as DG, diffusion_oracle, reflow_oracle
    dev = torch.device("cuda:0")
    if kind == "wavenet":
        eager = reflow_oracle.seeded_weights(diffusion_oracle.WaveNet(M, 20, 512, 256), 5)
        net = pkg.WaveNet(M, 20, 512, 256)
        net.diffusion_backward = True
        Mc = 256
    else:
        eager = reflow_oracle.seeded_weights(reflow_oracle.VelocityNet(M, 512, 128, 6), 5)
        net = pkg.NaiveV2Diff(mel_channels=M, dim=512, num_layers=6, condition_dim=128, use_mlp=False)
        net.reflow_backward = True
        Mc = 128
    net.load_state_dict(eager.state_dict(), strict=True)
    diff = pkg.GaussianDiffusion(net.to(dev), out_dims=M).to(dev).train()
    eager = eager.to(dev).train()
    g = torch.Generator().manual_seed(B * T)
    ramp = lambda n: torch.linspace(-8.0, 0.5, n)[None, None, :]
    cond = (ramp(Mc) + 1.5 * torch.randn(B, T, Mc, generator=g)).to(dev)
    gt = (ramp(M) + 1.5 * torch.randn(B, T, M, generator=g)).to(dev)
    torch.manual_seed(1)
    t, noise = DG.draws(B, T, t_max, device=dev)
    cg = cond.clone().requires_grad_(True)
    k_loss = lambda: diff._loss(cg, gt, t, noise)
    e_loss = lambda: DG.oracle_loss(eager, cg, gt, t, noise)

    def clear():
        diff.zero_grad(set_to_none=True)
        eager.zero_grad(set_to_none=True)
        cg.grad = None

    res = {"B": B, "frames": T, "denoiser": kind, "t_max": t_max}
    res["loss_forward_ms"], res["loss_forward_eager_ms"], sa, sb = alternate(k_loss, e_loss, clear, flush, steps, warmup)
    res["loss_fwd_bwd_ms"], res["loss_fwd_bwd_eager_ms"], sc, sd = alternate(lambda: k_loss().backward(),
                                                                            lambda: e_loss().backward(), clear, flush,
                                                                            steps, warmup)
    res["spreads_ms"] = {"loss_forward": sa, "loss_forward_eager": sb, "loss_fwd_bwd": sc, "loss_fwd_bwd_eager": sd}
    res["loss_fwd_bwd_speedup"] = res["loss_fwd_bwd_eager_ms"] / res["loss_fwd_bwd_ms"]
    fwd, bwd = gemm_flop(kind, B, T)
    res["gemm_gflop_forward"], res["gemm_gflop_backward"] = fwd / 1e9, bwd / 1e9
    res["kernels_gemm_tflops_fwd_bwd"] = (fwd + bwd) / (res["loss_fwd_bwd_ms"] * 1e-3) / 1e12
    with torch.no_grad():
        base_k, base_e = held(k_loss), held(e_loss)
    res["saved_activations_mb"] = (held(k_loss) - base_k) / 2 ** 20
    res["saved_activations_eager_mb"] = (held(e_loss) - base_e) / 2 ** 20
    clear()
    torch.cuda.reset_peak_memory_stats()
    k_loss().backward()
    torch.cuda.synchronize()
    res["peak_allocated_fwd_bwd_mb"] = torch.cuda.max_memory_allocated() / 2 ** 20
    clear()
    torch.cuda.reset_peak_memory_stats()
    e_loss().backward()
    torch.cuda.synchronize()
    res["peak_allocated_fwd_bwd_eager_mb"] = torch.cuda.max_memory_allocated() / 2 ** 20
    clear()
    with torch.no_grad():
        lk, le = k_loss(), e_loss()
    res["loss_rel_diff_kernels_vs_eager"] = abs(lk.item() - le.item()) / abs(le.item())
    del diff, eager
    torch.cuda.empty_cache()
    return {k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}


def run_step(B, T, flush, steps, warmup):
    import torch
    import ddsp_svc_b200 as pkg
    from ddsp_svc_b200 import mel as pm, synthetic as syn
    from tests import diffusion_grad_oracle as DG, diffusion_oracle, reflow_oracle
    from tests.u2c_pcmer_oracle import PCmerUnit2Control
    SR, P, N_UNIT = 44100, 512, 768
    dev = torch.device("cuda:0")
    torch.manual_seed(2)
    ours = pkg.CombSubFast(SR, P, n_unit=N_UNIT, n_spk=2, use_pitch_aug=True)
    ours.unit2ctrl.pcmer_backward = True
    ours = ours.to(dev).train()
    u2c_eager = PCmerUnit2Control(N_UNIT, 2, ours.unit2ctrl.output_splits, use_pitch_aug=True).train()
    u2c_eager.load_state_dict(ours.unit2ctrl.state_dict())
    theirs = pkg.CombSubFast(SR, P, unit2ctrl=u2c_eager).to(dev).train()
    wn_eager = reflow_oracle.seeded_weights(diffusion_oracle.WaveNet(M, 20, 512, 256), 5)
    net = pkg.WaveNet(M, 20, 512, 256)
    net.load_state_dict(wn_eager.state_dict(), strict=True)
    net.diffusion_backward = True
    diff = pkg.GaussianDiffusion(net.to(dev), out_dims=M).to(dev).train()
    wn_eager = wn_eager.to(dev).train()
    stft = pm.STFT(SR, M, 2048, 2048, P, 40, 16000)
    g = torch.Generator().manual_seed(B * T + 1)
    units, volume = torch.randn(B, T, N_UNIT, generator=g).to(dev), (0.2 * torch.rand(B, T, 1, generator=g)).to(dev)
    f0 = syn.make_f0(B, T, SR, P).to(dev)
    spk, aug = torch.randint(1, 3, (B, 1), generator=g).to(dev), torch.randn(B, 1, 1, generator=g).to(dev)
    with torch.no_grad():
        sig, _, _ = ours(units, f0, volume, spk_id=spk, aug_shift=aug)
        mel0 = stft.get_mel(sig).transpose(1, 2)
        gt = (mel0 + 0.5 * torch.randn_like(mel0)).contiguous()

    def step_of(model, diffusion_loss):
        def step():
            signal, hidden, _ = model(units, f0, volume, spk_id=spk, aug_shift=aug, infer=False)
            mel = stft.get_mel(signal).transpose(1, 2)
            torch.manual_seed(3)
            t, noise = DG.draws(B, T, 100, device=dev)
            (torch.nn.functional.mse_loss(mel, gt) + diffusion_loss(hidden, t, noise)).backward()
        return step

    def clear():
        for m in (ours, theirs, diff, wn_eager):
            m.zero_grad(set_to_none=True)

    a = step_of(ours, lambda h, t, noise: diff._loss(h, gt, t, noise))
    b = step_of(theirs, lambda h, t, noise: DG.oracle_loss(wn_eager, h, gt, t, noise))
    res = {"B": B, "frames": T}
    res["step_ms"], res["step_eager_ms"], sa, sb = alternate(a, b, clear, flush, steps, warmup)
    res["spreads_ms"] = {"step": sa, "step_eager": sb}
    res["step_speedup"] = res["step_eager_ms"] / res["step_ms"]
    del ours, theirs, diff, wn_eager
    torch.cuda.empty_cache()
    return {k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed calls per arm and row")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_diffusion_grad.py needs a CUDA device (no fallback)")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    res = {"bench": "diffusion_train_loss", "card": card(), "gemm_precision": "3xtf32 (default)",
           "timing": "median of %d calls per arm after %d warm-up calls, arms alternating, CUDA events, L2 flushed before "
                     "each call (untimed); eager arm: plain-torch networks in fp32 under torch's defaults"
                     % (args.steps, args.warmup),
           "rows": {label: run_row(kind, B, T, t_max, flush, args.steps, args.warmup) for label, kind, B, T, t_max in ROWS},
           "steps": {label: run_step(B, T, flush, args.steps, args.warmup) for label, B, T in STEP_ROWS}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
