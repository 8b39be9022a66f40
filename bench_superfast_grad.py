"""Training step of CombSubSuperFast's DSP on the kernels: forward, backward and forward + backward per step, and the
same step done by the reference's algorithm (oracle port under autograd) eagerly on the same GPU.  Prints one JSON line.

    python bench_superfast_grad.py [--steps 20] [--warmup 3]

Shapes: the training batch of configs/combsub.yaml (24 x 2 s, 172 frames) and BASELINE config 3 (32 x 10 s).
Every step is timed with CUDA events after the L2 was flushed (256 MiB memset, untimed); the medians are reported.
The backward's bytes/s counts the four controls read, the four gradients written and dL/dsignal read.
Needs a CUDA device; there is no fallback."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SR, P, WIN = 44100, 512, 2048
NB = WIN // 2 + 1
SHAPES = [("combsub_yaml_train_b24_2s", 24, 172), ("baseline_cfg3_b32_10s", 32, 861)]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=power.limit,power.max_limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        limit, max_limit = float(q[0]), float(q[1])
    except Exception:
        limit = max_limit = None
    return {"name": name, "power_limit_w": limit, "power_max_limit_w": max_limit}


def timed(fn, prep, flush, steps, warmup):
    import torch
    for _ in range(warmup):
        prep()
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        prep()
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def run_shape(label, B, nF, flush, steps, warmup):
    import torch
    from ddsp_svc_b200 import ops, synthetic as syn
    from oracle import torch_port as tp
    dev = torch.device("cuda", torch.cuda.current_device())
    sm = syn.superfast_split_map(WIN)
    f0 = syn.make_f0(B, nF, SR, P).to(dev)
    dense, _ = syn.make_ctrl(B, nF, sm)
    leaf = dense.to(dev).requires_grad_(True)
    cot = torch.randn(B, nF * P, generator=torch.Generator().manual_seed(1)).to(dev)
    st = {}

    def fwd():
        ws, _ = ops.superfast_scan(f0, P, SR)
        c = syn.split_views(leaf, sm)
        st["sig"] = ops.superfast_synth(ws, c["harmonic_magnitude"], c["harmonic_phase"], c["noise_magnitude"],
                                        c["noise_phase"], P, WIN, seed=7)

    def bwd():
        st["sig"].backward(cot)

    def clear():
        leaf.grad = None

    def prep_bwd():
        clear()
        fwd()

    fwd_ms = timed(fwd, clear, flush, steps, warmup)
    bwd_ms = timed(bwd, prep_bwd, flush, steps, warmup)
    step_ms = timed(lambda: (fwd(), bwd()), clear, flush, steps, warmup)
    # the backward kernel alone (what the bytes/s refers to)
    ws, _ = ops.superfast_scan(f0, P, SR)
    c = syn.split_views(leaf.detach(), sm)
    kern = lambda: ops.superfast_synth_backward(ws, c["harmonic_magnitude"], c["harmonic_phase"], c["noise_magnitude"],
                                                c["noise_phase"], cot, P, WIN, seed=7)
    kern_ms = timed(kern, lambda: None, flush, steps, warmup)
    nbytes = 4 * (2 * 4 * B * nF * NB + B * nF * P)
    st.clear()
    torch.cuda.empty_cache()

    # the reference's algorithm under autograd, eagerly on this GPU (every tensor the port creates lands on the device)
    pleaf = dense.to(dev).requires_grad_(True)
    noise = torch.randn(B, nF * P, device=dev)

    def port_step():
        with torch.device(dev):
            out = tp.superfast_forward(f0, syn.split_views(pleaf, sm), SR, P, WIN, noise=noise)["signal"]
        out.backward(cot)

    def port_prep():
        pleaf.grad = None
    port_ms = timed(port_step, port_prep, flush, max(3, steps // 4), 1)
    del pleaf, noise
    torch.cuda.empty_cache()
    return {"B": B, "n_frames": nF, "seconds": nF * P / SR,
            "forward_ms": fwd_ms, "backward_ms": bwd_ms, "forward_backward_ms": step_ms,
            "backward_kernel_ms": kern_ms, "backward_kernel_bytes": nbytes,
            "backward_kernel_GBps": nbytes / (kern_ms * 1e-3) / 1e9,
            "port_eager_forward_backward_ms": port_ms, "speedup_vs_port": port_ms / step_ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_superfast_grad.py needs a CUDA device (no fallback)")
    from ddsp_svc_b200 import _lib
    _lib.lib()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    line = {"metric": "superfast_train_step", "card": card(),
            "timing": "median of %d steps after %d warm-up, CUDA events, L2 flushed before each step (untimed); "
                      "forward = frame scan + synthesis, backward = autograd backward (kernel + split into the dense "
                      "control gradient); port = oracle.torch_port.superfast_forward under autograd, eager, same GPU"
                      % (args.steps, args.warmup),
            "shapes": {label: run_shape(label, B, nF, flush, args.steps, args.warmup) for label, B, nF in SHAPES}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
