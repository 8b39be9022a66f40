"""The random-scale spectral loss of configs/combsub.yaml on the kernels (RSSLoss(256, 2048, 4), csrc/rss_loss.cu):
loss forward, loss backward, per-kernel times, and the whole training step CombSubSuperFast forward -> RSSLoss ->
backward through both, against the same loss / step done by the reference's algorithm (oracle.loss on torch.stft in
torchaudio's order, oracle port for the synthesizer) eagerly under autograd on the same GPU.  Prints one JSON line.

    python bench_rss_loss.py [--steps 20] [--warmup 3]

Shapes: the training batch of configs/combsub.yaml (24 x 2 s, 172 hops) and BASELINE config 3 (32 x 10 s).  Scales:
redrawn every step by RSSLoss itself from a seeded torch generator (the mix of Bluestein sizes 1024 / 2048 / 4096 that
training sees), and a fixed worst case of four scales of 2047 (all 4096-point transforms).  Every step is timed with
CUDA events after the L2 was flushed (256 MiB memset, untimed); the medians are reported.  Kernel times come from a
separate torch.profiler run.  FLOPs count 5 M log2 M per M-point complex FFT: 4 per frame in the forward (two Bluestein transforms, prediction
and target), 6 in the backward.  The per-n tables of the kernels (RSSLoss.prebuild_tables) and the eager side's
cuFFT plans of all 1792 sizes at the timed shape, forward and backward, are built before timing (the plan cache is
raised to 8192 entries so none is evicted; the JSON records how many it holds): both sides are timed warm, as after a
while of training.  Needs a CUDA device; there is no fallback."""
import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_superfast_grad import card, timed  # noqa: E402

SR, P, WIN = 44100, 512, 2048
SHAPES = [("combsub_yaml_train_b24_2s", 24, 172), ("baseline_cfg3_b32_10s", 32, 861)]
FFT_MIN, FFT_MAX, N_SCALE = 256, 2048, 4


def fft_flops(B, T, n_ffts, per_frame):
    import math
    from ddsp_svc_b200.loss import bluestein_size
    total = 0
    for n in n_ffts:
        M = bluestein_size(n)
        frames = B * (1 + (T - n) // n)
        total += frames * per_frame * 5 * M * math.log2(M)
    return total


def kernel_times(fn, steps):
    """mean device time per call of every rss_* kernel over ``steps`` calls (torch.profiler, CUDA activity)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "rss_" in ev.key:
            m = re.search(r"rss_\w+?_kernel(<\d+>)?", ev.key)
            name = m.group(0) if m else ev.key
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            out[name] = out.get(name, 0.0) + t / 1e3 / steps
    return out


def run_shape(B, nF, flush, steps, warmup):
    import torch
    from ddsp_svc_b200 import CombSubSuperFast, FixedControls, RSSLoss, synthetic as syn
    from oracle import loss as ol, torch_port as tp
    dev = torch.device("cuda", torch.cuda.current_device())
    sm = syn.superfast_split_map(WIN)
    f0 = syn.make_f0(B, nF, SR, P).to(dev)
    dense, _ = syn.make_ctrl(B, nF, sm)
    teacher, _ = syn.make_ctrl(B, nF, sm, seed=8)
    leaf = dense.to(dev).requires_grad_(True)
    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=FixedControls(syn.split_views(leaf, sm),
                                                                  torch.zeros(B, nF, 256, device=dev))).to(dev)
    T = nF * P
    with torch.no_grad():
        y = model(None, f0, None)[0]
        target = CombSubSuperFast(SR, P, WIN, unit2ctrl=FixedControls(syn.split_views(teacher.to(dev), sm), None)).to(dev)(
            None, f0, None)[0]
    crit = RSSLoss(FFT_MIN, FFT_MAX, N_SCALE)
    crit.prebuild_tables(dev)
    yg = y.clone().requires_grad_(True)
    # the eager side's cuFFT plans of every size at the timed shape, forward and backward (the plan cache keys on the
    # batch too), as after a while of training; the cache is sized so that none is evicted
    cache = torch.backends.cuda.cufft_plan_cache[dev.index]
    cache.max_size = max(cache.max_size, 8192)
    yw = y.clone().requires_grad_(True)
    for n in range(FFT_MIN, FFT_MAX):
        ol.rss_loss(yw, target, [n]).backward()
    torch.cuda.synchronize()
    plans = cache.size
    del yw
    out = {"B": B, "n_frames": nF, "seconds": T / SR, "eager_cufft_plans_cached": plans,
           "eager_cufft_plan_cache_max": cache.max_size}
    for label, pinned in (("random_scales", None), ("all_2047", [2047] * N_SCALE)):
        torch.manual_seed(0)
        draws = [torch.randint(FFT_MIN, FFT_MAX, (N_SCALE,)).tolist() for _ in range(64)]
        mean_flops_f = sum(fft_flops(B, T, d, 4) for d in draws) / len(draws) if pinned is None else fft_flops(B, T, pinned, 4)
        mean_flops_b = sum(fft_flops(B, T, d, 6) for d in draws) / len(draws) if pinned is None else fft_flops(B, T, pinned, 6)
        torch.manual_seed(0)

        def fwd():
            with torch.no_grad():
                crit(y, target, n_ffts=pinned)

        def fwd_bwd():
            crit(yg, target, n_ffts=pinned).backward()

        def clear():
            yg.grad = None

        def step():
            signal, _, _ = model(None, f0, None, infer=False)
            crit(signal, target, n_ffts=pinned).backward()

        def clear_step():
            leaf.grad = None

        f_ms = timed(fwd, lambda: None, flush, steps, warmup)
        fb_ms = timed(fwd_bwd, clear, flush, steps, warmup)
        step_ms = timed(step, clear_step, flush, steps, warmup)
        torch.manual_seed(0)
        kern = kernel_times(fwd_bwd, max(5, steps // 2))

        # the reference's algorithm under autograd, eagerly on this GPU (same scale draws)
        pleaf = dense.to(dev).requires_grad_(True)
        noise = torch.randn(B, T, device=dev)
        ygr = y.clone().requires_grad_(True)

        def draw():
            return pinned if pinned is not None else torch.randint(FFT_MIN, FFT_MAX, (N_SCALE,)).tolist()

        def ref_loss():
            ol.rss_loss(ygr, target, draw()).backward()

        def ref_step():
            with torch.device(dev):
                sig = tp.superfast_forward(f0, syn.split_views(pleaf, sm), SR, P, WIN, noise=noise)["signal"]
            ol.rss_loss(sig, target, draw()).backward()

        def ref_clear():
            pleaf.grad = None
            ygr.grad = None
        torch.manual_seed(0)
        ref_loss_ms = timed(ref_loss, ref_clear, flush, steps, warmup)
        torch.manual_seed(0)
        ref_step_ms = timed(ref_step, ref_clear, flush, max(3, steps // 4), 1)
        del pleaf, noise, ygr
        torch.cuda.empty_cache()
        bwd_ms = fb_ms - f_ms
        out[label] = {
            "loss_forward_ms": f_ms, "loss_forward_backward_ms": fb_ms, "loss_backward_ms": bwd_ms,
            "kernel_ms_per_call": kern,
            "forward_fft_gflop": mean_flops_f / 1e9, "forward_fft_tflops": mean_flops_f / (f_ms * 1e-3) / 1e12,
            "backward_fft_gflop": mean_flops_b / 1e9,
            "backward_fft_tflops": mean_flops_b / (bwd_ms * 1e-3) / 1e12 if bwd_ms > 0 else None,
            "reference_eager_loss_forward_backward_ms": ref_loss_ms,
            "loss_speedup_vs_reference": ref_loss_ms / fb_ms,
            "train_step_ms": step_ms, "reference_eager_train_step_ms": ref_step_ms,
            "step_speedup_vs_reference": ref_step_ms / step_ms}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_rss_loss.py needs a CUDA device (no fallback)")
    from ddsp_svc_b200 import _lib
    _lib.lib()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    line = {"metric": "rss_loss_train_step", "card": card(),
            "timing": "median of %d steps after %d warm-up, CUDA events, L2 flushed before each step (untimed); "
                      "loss = RSSLoss(256, 2048, 4) forward (+ backward); step = superfast frame scan + synthesis + "
                      "loss + autograd backward through both; reference = oracle.loss (torch.stft, torchaudio's order) "
                      "+ oracle.torch_port.superfast_forward under autograd, eager, same GPU" % (args.steps, args.warmup),
            "shapes": {label: run_shape(B, nF, flush, args.steps, args.warmup) for label, B, nF in SHAPES}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
