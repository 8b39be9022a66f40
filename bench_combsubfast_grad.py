"""Training step of CombSubFast's DSP on the kernels (infer=False): forward, the backward kernel, forward + backward and
the DiffusionNew DDSP-loss step, and the same steps done by the reference's algorithm (oracle port under autograd)
eagerly on the same GPU.  Prints one JSON line.

    python bench_combsubfast_grad.py [--steps 20] [--warmup 3]

Shapes: the training batch of configs/diffusion-new.yaml (36 x 2 s, 172 frames) and 32 x 10 s.
Every step is timed with CUDA events after the L2 was flushed (256 MiB memset, untimed); the medians are reported.
The backward kernel's bytes/s counts the comb, the three controls and dL/dsignal read and the three gradients written
(the in-kernel noise is generated, not read).
The DDSP-loss step is diffusion/vocoder.py:246-253: synthesizer -> get_mel -> transpose -> mse_loss -> backward.
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

SR, P = 44100, 512
NB = P + 1
SHAPES = [("diffusion_new_train_b36_2s", 36, 172), ("b32_10s", 32, 861)]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=power.limit,power.max_limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        limit, max_limit, sm_clock = float(q[0]), float(q[1]), float(q[2])
    except Exception:
        limit = max_limit = sm_clock = None
    return {"name": name, "power_limit_w": limit, "power_max_limit_w": max_limit, "max_sm_clock_mhz": sm_clock}


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


def eager_mel(y, basis):
    """oracle.mel.get_mel (keyshift 0, speed 1) on the tensor's device: the reference's torch operators"""
    import torch
    import torch.nn.functional as F
    window = torch.hann_window(2048, device=y.device)
    y = F.pad(y.unsqueeze(1), (768, 768), mode="reflect").squeeze(1)
    spec = torch.stft(y, 2048, hop_length=512, win_length=2048, window=window, center=False, pad_mode="reflect",
                      normalized=False, onesided=True, return_complex=True)
    spec = torch.sqrt(spec.real.pow(2) + spec.imag.pow(2) + (1e-9))
    return torch.log(torch.clamp(torch.matmul(basis, spec), min=1e-5))


def run_shape(B, nF, flush, steps, warmup):
    import torch
    from ddsp_svc_b200 import CombSubFast, FixedControls, ops, synthetic as syn
    from ddsp_svc_b200 import mel as pm
    from oracle import mel as om
    from oracle import torch_port as tp
    dev = torch.device("cuda", torch.cuda.current_device())
    sm = syn.combsubfast_split_map(P)
    f0 = syn.make_f0(B, nF, SR, P).to(dev)
    dense, _ = syn.make_ctrl(B, nF, sm)
    leaf = dense.to(dev).requires_grad_(True)
    model = CombSubFast(SR, P, unit2ctrl=FixedControls(syn.split_views(leaf, sm), None)).to(dev)
    cot = torch.randn(B, nF * P, generator=torch.Generator().manual_seed(1)).to(dev)
    stft = pm.STFT(SR, 128, 2048, 2048, 512, 40, 16000)
    st = {}

    def fwd():
        st["sig"] = model(None, f0, None, infer=False)[0]

    def bwd():
        st["sig"].backward(cot)

    def clear():
        leaf.grad = None

    def prep_bwd():
        clear()
        fwd()

    with torch.no_grad():
        gt_spec = stft.get_mel(model(None, f0, None, infer=False)[0]).transpose(1, 2) + 0.1

    def ddsp_step():
        sig = model(None, f0, None, infer=False)[0]
        torch.nn.functional.mse_loss(stft.get_mel(sig).transpose(1, 2), gt_spec).backward()

    fwd_ms = timed(fwd, clear, flush, steps, warmup)
    bwd_ms = timed(bwd, prep_bwd, flush, steps, warmup)
    step_ms = timed(lambda: (fwd(), bwd()), clear, flush, steps, warmup)
    ddsp_ms = timed(ddsp_step, clear, flush, steps, warmup)
    # the backward kernel alone (what the bytes/s refers to)
    fp, _ = ops.phase_scan(f0, P, SR, None, False)
    comb = ops.comb_source(f0, fp, P, SR, infer=False)
    c = syn.split_views(leaf.detach(), sm)
    kern = lambda: ops.combsubfast_filter_backward(comb, c["harmonic_magnitude"], c["harmonic_phase"],
                                                   c["noise_magnitude"], cot, P, seed=7)
    kern_ms = timed(kern, lambda: None, flush, steps, warmup)
    nbytes = 4 * (2 * 3 * B * nF * NB + 2 * B * nF * P)
    st.clear()
    torch.cuda.empty_cache()

    # the reference's algorithm under autograd, eagerly on this GPU (every tensor the port creates lands on the device)
    pleaf = dense.to(dev).requires_grad_(True)
    noise = torch.rand(B, nF * P, device=dev) * 2 - 1
    basis = torch.from_numpy(om.librosa_mel(sr=SR, n_fft=2048, n_mels=128, fmin=40, fmax=16000)).float().to(dev)

    def port_signal():
        with torch.device(dev):
            return tp.combsubfast_forward(f0, syn.split_views(pleaf, sm), SR, P, noise=noise, infer=False)["signal"]

    def port_step():
        port_signal().backward(cot)

    def port_ddsp_step():
        sig = port_signal()
        torch.nn.functional.mse_loss(eager_mel(sig, basis).transpose(1, 2), gt_spec).backward()

    def port_prep():
        pleaf.grad = None
    port_ms = timed(port_step, port_prep, flush, max(3, steps // 4), 1)
    port_ddsp_ms = timed(port_ddsp_step, port_prep, flush, max(3, steps // 4), 1)
    del pleaf, noise
    torch.cuda.empty_cache()
    return {"B": B, "n_frames": nF, "seconds": nF * P / SR,
            "forward_ms": fwd_ms, "backward_ms": bwd_ms, "forward_backward_ms": step_ms,
            "backward_kernel_ms": kern_ms, "backward_kernel_bytes": nbytes,
            "backward_kernel_GBps": nbytes / (kern_ms * 1e-3) / 1e9,
            "ddsp_loss_step_ms": ddsp_ms,
            "port_eager_forward_backward_ms": port_ms, "port_eager_ddsp_loss_step_ms": port_ddsp_ms,
            "speedup_vs_port": port_ms / step_ms, "ddsp_loss_speedup_vs_port": port_ddsp_ms / ddsp_ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_combsubfast_grad.py needs a CUDA device (no fallback)")
    from ddsp_svc_b200 import _lib
    _lib.lib()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    line = {"metric": "combsubfast_train_step", "card": card(),
            "timing": "median of %d steps after %d warm-up, CUDA events, L2 flushed before each step (untimed); "
                      "forward = phase scan + comb source + filter, backward = autograd backward (kernel + split into "
                      "the dense control gradient); ddsp loss = forward + get_mel + mse_loss + backward; port = "
                      "oracle.torch_port.combsubfast_forward (+ the reference's mel on torch) under autograd, eager, "
                      "same GPU" % (args.steps, args.warmup),
            "shapes": {label: run_shape(B, nF, flush, args.steps, args.warmup) for label, B, nF in SHAPES}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
