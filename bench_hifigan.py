"""Time the NSF-HiFiGAN generator (ddsp_svc_b200.Generator) of the 44.1 kHz, 128-bin, hop-512 vocoder against the same
network written in plain torch (tests/hifigan_oracle.py) run eagerly in fp32 on the same GPU under torch's defaults --
cuDNN convolutions in TF32, what the reference runs today.  Both arms get the same harmonic source: the kernels' arm
computes it (the fused SourceModuleHnNSF kernel is part of its forward), the eager arm is handed it precomputed.

    python bench_hifigan.py [--steps K] [--warmup W]

Shapes: 1 x 172 frames (the 2 s slices gui.py and main.py enhance), 1 x 861 (a 10 s slice of main_diff.py) and
16 x 861.  The two arms alternate call by call; each call is timed with CUDA events after the L2 was flushed (256 MiB
memset, untimed); medians of K calls per arm after W warm-up calls of each.  Also reported: kernel launches per call and
per-stage kernel times (both from torch.profiler in a separate untimed call), the GFLOP of one call from shapes and the
rate it implies ("fp32-grade": 3xTF32 products, each counted once).  Prints one JSON line, with the card's name and
power limit read in the same run.  Writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import warnings

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_reflow import card, one  # noqa: E402

SHAPES = [("1x172", 1, 172), ("1x861", 1, 861), ("16x861", 16, 861)]


def gflop(h, B, nF):
    """multiply-adds x 2 of one call: conv_pre, per stage the transposed convolution (C_in C_out 2u per input frame),
    the noise convolution and 3 x 6 resblock convolutions, conv_post"""
    T, C = nF, h["upsample_initial_channel"]
    f = 2 * B * nF * h["num_mels"] * C * 7
    rates = h["upsample_rates"]
    for i, u in enumerate(rates):
        f += 2 * B * T * C * (C // 2) * 2 * u
        T, C = T * u, C // 2
        s = 1
        for r in rates[i + 1:]:
            s *= r
        f += 2 * B * T * C * (2 * s if i + 1 < len(rates) else 1)
        f += 2 * B * T * C * C * 6 * sum(h["resblock_kernel_sizes"])
    f += 2 * B * T * C * 7
    return f / 1e9


def stage_times(fn, n_stages):
    """torch.profiler kernel times of one call, grouped by position in launch order: source, conv_pre, each stage's
    transposed convolution + 18 resblock convolutions, post (ms); and the number of kernels"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                key=lambda e: e.time_range.start)
    us = [e.time_range.end - e.time_range.start for e in ev]
    groups = {"source": us[:2], "conv_pre": us[2:3]}
    for i in range(n_stages):
        groups["stage%d" % i] = us[3 + 19 * i:3 + 19 * (i + 1)]
    groups["post"] = us[3 + 19 * n_stages:]
    return {k: round(sum(v) / 1e3, 4) for k, v in groups.items()}, len(ev)


def run_shape(B, nF, flush, reps, warmup):
    import torch
    import ddsp_svc_b200 as pkg
    from tests import hifigan_oracle as ho
    from tests.golden import make_golden_hifigan as mk
    dev = torch.device("cuda:0")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen = pkg.Generator(ho.config(ho.FULL))
    sd = mk.seeded_state_dict("full")
    gen.load_state_dict(sd, strict=True)
    gen.remove_weight_norm()
    gen = gen.to(dev).eval()
    eager = ho.build(ho.config(ho.FULL), sd, torch.float32).to(dev)
    g = torch.Generator().manual_seed(B * nF)
    x = (torch.linspace(-8.0, 0.5, 128)[None, :, None] + 1.5 * torch.randn(B, 128, nF, generator=g)).to(dev)
    f0 = (100.0 + 300.0 * torch.rand(B, nF, generator=g)).to(dev)
    noise = torch.randn(B, nF * 512, 9, generator=g).to(dev)
    rand_ini = torch.rand(1, 1, 9, generator=g).to(dev)
    rand_ini[..., 0] = 0
    xv = x.transpose(1, 2).contiguous().transpose(1, 2)        # NsfHifiGAN's mel.transpose(1, 2) view
    kern = lambda: gen(xv, f0, rand_ini, noise)
    with torch.no_grad():
        har = gen.m_source(f0, gen.upp, rand_ini, noise)
        ref = lambda: eager(xv, har)
        for _ in range(warmup):
            kern()
            ref()
        ta, tb = [], []
        for _ in range(reps):
            ta.append(one(kern, flush))
            tb.append(one(ref, flush))
        out_k, out_r = kern(), ref()
        stages, n_launch = stage_times(kern, len(ho.FULL["upsample_rates"]))
    k_ms, r_ms = statistics.median(ta), statistics.median(tb)
    gf = gflop(ho.FULL, B, nF)
    return {"B": B, "frames": nF, "samples": nF * 512, "kernels_ms": round(k_ms, 3), "eager_fp32_ms": round(r_ms, 3),
            "speedup_vs_eager": round(r_ms / k_ms, 3),
            "kernels_ms_spread": [round(min(ta), 3), round(max(ta), 3)], "eager_ms_spread": [round(min(tb), 3), round(max(tb), 3)],
            "launches_per_call": n_launch, "gflop": round(gf, 2), "kernels_tflops_fp32_grade": round(gf / k_ms, 2),
            "eager_tflops": round(gf / r_ms, 2), "stage_kernel_ms": stages,
            "rel_rms_kernels_vs_eager": float((out_k - out_r).pow(2).mean().sqrt() / out_r.pow(2).mean().sqrt())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed calls per arm and shape")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_hifigan.py needs a CUDA device")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    res = {"bench": "nsf_hifigan_generator", "card": card(), "precision": "3xTF32 tensor cores; eager arm fp32 (cuDNN TF32)",
           "timing": "median of %d calls per arm after %d warm-up calls, arms alternating, CUDA events, L2 flushed before "
                     "each call (untimed)" % (args.steps, args.warmup),
           "shapes": {label: run_shape(B, nF, flush, args.steps, args.warmup) for label, B, nF in SHAPES}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
