"""Time the diffusion models' sampler (ddsp_svc_b200.GaussianDiffusion around WaveNet(128, 20, 512, 256) of
configs/diffusion-new.yaml, and around NaiveV2Diff(dim 512, 6 layers) of configs/diffusion-fast.yaml) against the same
sampler written in plain torch (tests/diffusion_oracle.py) run eagerly in fp32 on the same GPU under torch's defaults --
cuDNN convolutions in TF32, what the reference runs today.

    python bench_diffusion.py [--steps K] [--warmup W]

Shapes: one 10 s slice of main_diff.py (1 x 861 frames) with dpm-solver from k_step 100 at speedup 10 (10 network
evaluations) and with DDPM from k_step 100 (100 evaluations), 16 slices x 861 frames with dpm-solver, and the
diffusion-fast.yaml denoiser on one slice with dpm-solver; the shallow start from a DDSP mel, as Unit2Wav samples.  DDPM's
per-step noise is drawn once, outside the timed calls, and fed to both arms.  The two arms alternate call by call; each
call is timed with CUDA events after the L2 was flushed (256 MiB memset, untimed); medians of K calls per arm after W
warm-up calls of each.  Also reported: kernel launches per network evaluation (counted with torch.profiler in a separate
untimed call) and the GEMM FLOP per evaluation and per call from shapes.  Prints one JSON line, with the card's name and
power limit read in the same run.  Writes nothing.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_reflow import card, launches, one  # noqa: E402

M, C, LAYERS, HIDDEN = 128, 512, 20, 256          # diffusion-new.yaml's WaveNet
FAST_DIM, FAST_LAYERS = 512, 6                    # diffusion-fast.yaml's NaiveV2Diff (condition: the 128-bin mel)
SHAPES = [("new_1x861_dpm10", "wavenet", 1, 861, "dpm-solver", 10), ("new_1x861_ddpm100", "wavenet", 1, 861, None, 1),
          ("new_16x861_dpm10", "wavenet", 16, 861, "dpm-solver", 10), ("fast_1x861_dpm10", "naive", 1, 861, "dpm-solver", 10)]


def gemm_flop(kind, B, T):
    """(multiply-adds x 2 of one network evaluation, of the once-per-call condition projections).  WaveNet per layer:
    the k = 3 convolution C -> 2 C (6 N C^2) and the output projection C -> 2 C (2 N C^2), 16 N C^2 FLOP; plus the input,
    skip and output projections.  NaiveV2Diff per layer: dim -> 4 dim and 2 dim -> dim."""
    N = B * T
    if kind == "wavenet":
        return 2 * N * (M * C + LAYERS * 8 * C * C + C * C + C * M), 2 * N * HIDDEN * LAYERS * 2 * C
    D = FAST_DIM
    return 2 * N * (M * D + FAST_LAYERS * (D * 4 * D + 2 * D * D) + D * M), 2 * N * M * FAST_LAYERS * D


def models(kind, dev):
    import ddsp_svc_b200 as pkg
    from tests import diffusion_oracle, reflow_oracle
    if kind == "wavenet":
        ref = diffusion_oracle.seeded_weights(diffusion_oracle.WaveNet(M, LAYERS, C, HIDDEN), 32)
        net = pkg.WaveNet(M, LAYERS, C, HIDDEN)
    else:
        ref = reflow_oracle.seeded_weights(reflow_oracle.VelocityNet(M, FAST_DIM, M, FAST_LAYERS), 44)
        net = pkg.NaiveV2Diff(mel_channels=M, dim=FAST_DIM, num_layers=FAST_LAYERS, condition_dim=M, use_mlp=False)
    net.load_state_dict(ref.state_dict(), strict=True)
    return pkg.GaussianDiffusion(net.to(dev).eval(), out_dims=M).to(dev), ref.to(dev).eval()


def run_shape(kind, B, T, method, speedup, flush, reps, warmup):
    import torch
    from tests import diffusion_oracle
    dev = torch.device("cuda:0")
    gd, eager = models(kind, dev)
    g = torch.Generator().manual_seed(B * T)
    ramp = lambda n: torch.linspace(-8.0, 0.5, n)[None, None, :]
    Mc = HIDDEN if kind == "wavenet" else M
    cond = (ramp(Mc) + 1.5 * torch.randn(B, T, Mc, generator=g)).to(dev)
    gt = (ramp(M) + 1.5 * torch.randn(B, T, M, generator=g)).to(dev)
    noise = torch.randn(B, 1, M, T, generator=g).to(dev)
    steps = torch.randn(100, B, 1, M, T, generator=g).to(dev) if speedup == 1 else None
    kern = lambda: gd._sample(cond, noise, gt, 100, speedup, method, steps)
    ref = lambda: diffusion_oracle.sample(eager, cond, noise, gt, 100, speedup, method, steps)[0]
    with torch.no_grad():
        for _ in range(warmup):
            kern()
            ref()
        ta, tb = [], []
        for _ in range(reps):
            ta.append(one(kern, flush))
            tb.append(one(ref, flush))
        out_k, out_r = kern(), ref()
        n_launch = launches(kern)
    evals = 100 // speedup
    k_ms, r_ms = statistics.median(ta), statistics.median(tb)
    per_eval, per_call = gemm_flop(kind, B, T)
    flop = per_eval * evals + per_call
    return {"denoiser": kind, "B": B, "frames": T, "method": method or "ddpm", "k_step": 100, "speedup": speedup,
            "evaluations": evals, "kernels_ms": round(k_ms, 3), "eager_fp32_ms": round(r_ms, 3),
            "speedup_vs_eager": round(r_ms / k_ms, 3),
            "kernels_ms_spread": [round(min(ta), 3), round(max(ta), 3)], "eager_ms_spread": [round(min(tb), 3), round(max(tb), 3)],
            "launches_per_evaluation": round(n_launch / evals, 1), "gemm_gflop_per_evaluation": round(per_eval / 1e9, 3),
            "gemm_gflop_per_call_once": round(per_call / 1e9, 3),
            "kernels_gemm_tflops": round(flop / (k_ms * 1e-3) / 1e12, 2),
            "rel_rms_kernels_vs_eager": float((out_k - out_r).pow(2).mean().sqrt() / out_r.pow(2).mean().sqrt())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed calls per arm and shape")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_diffusion.py needs a CUDA device")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    res = {"bench": "diffusion_sampler", "card": card(), "gemm_precision": "3xtf32 (default)",
           "timing": "median of %d calls per arm after %d warm-up calls, arms alternating, CUDA events, L2 flushed before "
                     "each call (untimed)" % (args.steps, args.warmup),
           "shapes": {label: run_shape(kind, B, T, m, s, flush, args.steps, args.warmup)
                      for label, kind, B, T, m, s in SHAPES}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
