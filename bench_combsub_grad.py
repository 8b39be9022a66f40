"""Training step of the old CombSub's DSP (training phase, infer=False) on the kernels: forward, backward kernels,
forward + backward, and the train.py step (CombSub -> RSSLoss(256, 2048, 4) -> backward); each against the reference's
algorithm (oracle port + oracle.loss under autograd) eagerly on the same GPU.  Prints one JSON line.

    python bench_combsub_grad.py [--steps 20] [--warmup 3]

Shapes: a training batch of 24 x 2 s (172 frames) and 32 x 10 s, at n_mag 256 / 512 / 256 (group delay / harmonic
magnitude / noise magnitude).  Every step is timed with CUDA events after the L2 was flushed (256 MiB memset, untimed); the medians are
reported.  The loss scales are pinned to one draw per shape so both sides transform the same sizes.
Needs a CUDA device; there is no fallback."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_superfast_grad import card, timed  # noqa: E402

SR, P, MA, MH, MN = 44100, 512, 256, 512, 256
SHAPES = [("train_b24_2s", 24, 172), ("b32_10s", 32, 861)]


def sm_clock():
    """the SM clock now and its maximum (MHz), read in the same run as the timings"""
    import subprocess
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20)
        now, peak = (float(v) for v in q.stdout.strip().split(","))
    except Exception:
        now = peak = None
    return {"sm_clock_mhz": now, "sm_clock_max_mhz": peak}


def run_shape(B, nF, flush, steps, warmup):
    import torch
    from ddsp_svc_b200 import RSSLoss, ops, synthetic as syn
    from oracle import loss as oloss, torch_port as tp
    dev = torch.device("cuda", torch.cuda.current_device())
    sm = syn.combsub_split_map(MA, MH, MN)
    f0 = syn.make_f0(B, nF, SR, P).to(dev)
    dense, _ = syn.make_ctrl(B, nF, sm)
    leaf = dense.to(dev).requires_grad_(True)
    cot = torch.randn(B, nF * P, generator=torch.Generator().manual_seed(1)).to(dev)
    target = (torch.rand(B, nF * P, generator=torch.Generator().manual_seed(2)) * 0.02 - 0.01).to(dev)
    n_ffts = [int(n) for n in oloss.draw_scales(256, 2048, 4)]
    crit = RSSLoss(256, 2048, 4)
    crit.prebuild_tables(dev)
    st = {}

    def fwd():
        frame_phase, _ = ops.phase_scan(f0, P, SR, infer=False)
        c = syn.split_views(leaf, sm)
        st["sig"] = ops.combsub_synth(f0, frame_phase, c["group_delay"], c["harmonic_magnitude"], c["noise_magnitude"],
                                      P, SR, seed=7, infer=False)[0]

    def clear():
        leaf.grad = None

    def prep_bwd():
        clear()
        fwd()

    fwd_ms = timed(fwd, clear, flush, steps, warmup)
    bwd_ms = timed(lambda: st["sig"].backward(cot), prep_bwd, flush, steps, warmup)
    step_ms = timed(lambda: (fwd(), st["sig"].backward(cot)), clear, flush, steps, warmup)

    def yaml_step():
        fwd()
        crit(st["sig"], target, n_ffts=n_ffts).backward()
    yaml_ms = timed(yaml_step, clear, flush, steps, warmup)

    # the backward kernels alone, on the workspace of one forward
    with torch.no_grad():
        frame_phase, _ = ops.phase_scan(f0, P, SR, infer=False)
        c = syn.split_views(leaf.detach(), sm)
        _, _, _, ws = ops._combsub_synth(f0, frame_phase, c["group_delay"], c["harmonic_magnitude"],
                                         c["noise_magnitude"], P, SR, seed=7, infer=False)
    kern = lambda: ops.combsub_synth_backward(f0, c["group_delay"], c["harmonic_magnitude"], c["noise_magnitude"], ws,
                                              cot, P, SR, seed=7)
    kern_ms = timed(kern, lambda: None, flush, steps, warmup)
    st.clear()
    del ws
    torch.cuda.empty_cache()

    # the reference's algorithm under autograd, eagerly on this GPU (every tensor the port creates lands on the device)
    pleaf = dense.to(dev).requires_grad_(True)
    noise = torch.rand(B, nF * P, device=dev) * 2 - 1

    def port_sig():
        with torch.device(dev):
            return tp.combsub_forward(f0, syn.split_views(pleaf, sm), SR, P, noise=noise, infer=False)["signal"]

    def port_prep():
        pleaf.grad = None
    n_port = max(3, steps // 4)
    port_ms = timed(lambda: port_sig().backward(cot), port_prep, flush, n_port, 1)

    def port_yaml():
        with torch.device(dev):
            oloss.rss_loss(port_sig(), target, n_ffts).backward()
    port_yaml_ms = timed(port_yaml, port_prep, flush, n_port, 1)
    del pleaf, noise
    torch.cuda.empty_cache()
    return {"B": B, "n_frames": nF, "seconds": nF * P / SR, "rss_n_ffts": n_ffts,
            "forward_ms": fwd_ms, "backward_ms": bwd_ms, "backward_kernels_ms": kern_ms,
            "forward_backward_ms": step_ms, "port_eager_forward_backward_ms": port_ms,
            "speedup_vs_port": port_ms / step_ms,
            "backward_over_forward": bwd_ms / fwd_ms,
            "train_step_ms": yaml_ms, "port_eager_train_step_ms": port_yaml_ms,
            "train_step_speedup_vs_port": port_yaml_ms / yaml_ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_combsub_grad.py needs a CUDA device (no fallback)")
    from ddsp_svc_b200 import _lib
    _lib.lib()
    torch.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    line = {"metric": "combsub_train_step", "card": dict(card(), **sm_clock()),
            "timing": "median of %d steps after %d warm-up, CUDA events, L2 flushed before each step (untimed); "
                      "forward = phase scan + synthesis (infer=False), backward = autograd backward (kernels + split "
                      "into the control views), train_step = forward + RSSLoss(256, 2048, 4) + backward; port = "
                      "oracle.torch_port.combsub_forward (+ oracle.loss.rss_loss) under autograd, eager, same GPU"
                      % (args.steps, args.warmup),
            "shapes": {label: run_shape(B, nF, flush, args.steps, args.warmup) for label, B, nF in SHAPES}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
