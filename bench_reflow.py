"""Time the reflow model's rectified-flow sampler (ddsp_svc_b200.RectifiedFlow around NaiveV2Diff at configs/reflow.yaml's
width: 512 channels, 6 layers, 128 mel bins) against the same sampler written in plain torch (tests/reflow_oracle.py) run
eagerly in fp32 on the same GPU under torch's defaults -- cuDNN convolutions in TF32, what the reference runs today.

    python bench_reflow.py [--steps K] [--warmup W]

Shapes: one 10 s slice of main_reflow.py (1 x 861 frames) with 20 Euler steps (reflow.yaml's infer_step) and with 5 RK4
steps (the same 20 network evaluations), and 16 slices x 861 frames with 20 Euler steps; t_start 0.7 from a DDSP mel,
as Unit2Wav samples.  The two arms alternate call by call; each call is timed with CUDA events after the L2 was flushed
(256 MiB memset, untimed); medians of K calls per arm after W warm-up calls of each.  Also reported: kernel launches per
network evaluation (counted with torch.profiler in a separate untimed call) and the GEMM FLOP per evaluation from
shapes.  Prints one JSON line, with the card's name and power limit read in the same run.  Writes nothing.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

M, DIM, LAYERS = 128, 512, 6
SHAPES = [("slice_1x861_euler20", 1, 861, "euler", 20), ("slice_1x861_rk4_5", 1, 861, "rk4", 5),
          ("batch_16x861_euler20", 16, 861, "euler", 20)]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        limit, sm_clock = float(q[0]), float(q[1])
    except Exception:
        limit = sm_clock = None
    return {"name": name, "power_limit_w": limit, "max_sm_clock_mhz": sm_clock}


def one(fn, flush):
    import torch
    flush.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def gemm_flop_per_eval(B, T):
    """multiply-adds x 2 of one velocity evaluation: input projection, per layer dim -> 4 dim and 2 dim -> dim, output
    projection (the condition projections run once per call, not per evaluation)"""
    N = B * T
    return 2 * N * (M * DIM + LAYERS * (DIM * 4 * DIM + 2 * DIM * DIM) + DIM * M)


def launches(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def run_shape(label, B, T, method, steps, flush, reps, warmup):
    import torch
    import ddsp_svc_b200 as pkg
    from tests import reflow_oracle
    from tests.golden import make_golden_reflow as mk
    dev = torch.device("cuda:0")
    net = pkg.NaiveV2Diff(use_mlp=False, **mk.model_kwargs("w512"))
    net.load_state_dict(mk.build_oracle("w512").state_dict(), strict=True)
    flow = pkg.RectifiedFlow(net.to(dev).eval())
    eager = mk.build_oracle("w512").to(dev).eval()
    g = torch.Generator().manual_seed(B * T)
    ramp = torch.linspace(-8.0, 0.5, M)[None, None, :]
    cond = (ramp + 1.5 * torch.randn(B, T, M, generator=g)).to(dev)
    noise = torch.randn(B, 1, M, T, generator=g).to(dev)
    kern = lambda: flow._sample(cond, noise, cond, steps, method, 0.7)
    ref = lambda: reflow_oracle.sample(eager, cond, noise, cond, steps, method, 0.7)
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
    evals = steps * (1 if method == "euler" else 4)
    k_ms, r_ms = statistics.median(ta), statistics.median(tb)
    flop = gemm_flop_per_eval(B, T)
    return {"B": B, "frames": T, "method": method, "infer_step": steps, "evaluations": evals,
            "kernels_ms": round(k_ms, 3), "eager_fp32_ms": round(r_ms, 3), "speedup": round(r_ms / k_ms, 3),
            "kernels_ms_spread": [round(min(ta), 3), round(max(ta), 3)], "eager_ms_spread": [round(min(tb), 3), round(max(tb), 3)],
            "launches_per_evaluation": round(n_launch / evals, 1), "gemm_gflop_per_evaluation": round(flop / 1e9, 3),
            "kernels_gemm_tflops": round(flop * evals / (k_ms * 1e-3) / 1e12, 2),
            "rel_rms_kernels_vs_eager": float((out_k - out_r).pow(2).mean().sqrt() / out_r.pow(2).mean().sqrt())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed calls per arm and shape")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_reflow.py needs a CUDA device")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    res = {"bench": "reflow_sampler", "card": card(), "gemm_precision": "3xtf32 (default)",
           "timing": "median of %d calls per arm after %d warm-up calls, arms alternating, CUDA events, L2 flushed before "
                     "each call (untimed)" % (args.steps, args.warmup),
           "shapes": {label: run_shape(label, B, T, m, s, flush, args.steps, args.warmup) for label, B, T, m, s in SHAPES}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
