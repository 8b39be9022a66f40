"""The DDSP loss of the reflow / diffusion models on the kernels: mel forward, the mel backward kernel, and the whole
training step CombSubSuperFast -> get_mel -> MSE -> backward through both, against the same step done by the reference's
algorithm (oracle port + the mel operators of oracle/mel.py) eagerly under autograd on the same GPU.  Prints one JSON line.

    python bench_mel_grad.py [--steps 20] [--warmup 3]

Shapes: the batch of configs/reflow.yaml (48 x 2 s, 172 frames) and BASELINE config 3 (32 x 10 s, 861 frames).
Every step is timed with CUDA events after the L2 was flushed (256 MiB memset, untimed); the medians are reported.
The backward kernel's bytes/s counts the waveform read, dL/dmel read and dL/dy written once each.
Needs a CUDA device; there is no fallback."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_superfast_grad import card, timed  # noqa: E402

SR, P, WIN, N_MELS = 44100, 512, 2048, 128
SHAPES = [("reflow_yaml_b48_2s", 48, 172), ("baseline_cfg3_b32_10s", 32, 861)]


def reference_get_mel(y, basis, window, hop=P, clip_val=1e-5):
    """oracle.mel.get_mel (nvSTFT.py:97-115, keyshift 0) with its tables already on y's device"""
    import torch
    import torch.nn.functional as F
    T = y.size(-1)
    pad_left = (WIN - hop) // 2
    pad_right = max((WIN - hop + 1) // 2, WIN - T - pad_left)
    y = F.pad(y.unsqueeze(1), (pad_left, pad_right), mode="reflect" if pad_right < T else "constant").squeeze(1)
    spec = torch.stft(y, WIN, hop_length=hop, win_length=WIN, window=window, center=False, pad_mode="reflect",
                      normalized=False, onesided=True, return_complex=True)
    spec = torch.sqrt(spec.real.pow(2) + spec.imag.pow(2) + 1e-9)
    return torch.log(torch.clamp(torch.matmul(basis, spec), min=clip_val))


def run_shape(B, nF, flush, steps, warmup):
    import torch
    import torch.nn.functional as F
    from ddsp_svc_b200 import CombSubSuperFast, FixedControls, mel as pm, synthetic as syn
    from oracle import mel as om, torch_port as tp
    dev = torch.device("cuda", torch.cuda.current_device())
    sm = syn.superfast_split_map(WIN)
    f0 = syn.make_f0(B, nF, SR, P).to(dev)
    dense, _ = syn.make_ctrl(B, nF, sm)
    leaf = dense.to(dev).requires_grad_(True)
    st = pm.STFT(SR, N_MELS, WIN, WIN, P, 40, 16000)
    model = CombSubSuperFast(SR, P, WIN, unit2ctrl=FixedControls(syn.split_views(leaf, sm),
                                                                  torch.zeros(B, nF, 256, device=dev))).to(dev)
    T = nF * P
    with torch.no_grad():
        y = model(None, f0, None)[0]
        mel = st.get_mel(y)
    n_frames = mel.shape[2]
    target = (mel.transpose(1, 2) + 0.1 * torch.randn(B, n_frames, N_MELS, device=dev)).contiguous()
    cot = torch.randn(B, N_MELS, n_frames, device=dev)

    def mel_fwd():
        with torch.no_grad():
            st.get_mel(y)

    def step():
        signal, _, _ = model(None, f0, None, infer=False)
        ddsp_mel = st.get_mel(signal).transpose(1, 2)          # reflow/vocoder.py extract()
        F.mse_loss(ddsp_mel, target).backward()

    def clear():
        leaf.grad = None

    mel_ms = timed(mel_fwd, lambda: None, flush, steps, warmup)
    kern_ms = timed(lambda: st.get_mel_backward(y, cot), lambda: None, flush, steps, warmup)
    step_ms = timed(step, clear, flush, steps, warmup)
    nbytes = 4 * (2 * B * T + B * N_MELS * n_frames)
    torch.cuda.empty_cache()

    # the reference's algorithm under autograd, eagerly on this GPU
    basis = torch.from_numpy(om.librosa_mel(sr=SR, n_fft=WIN, n_mels=N_MELS, fmin=40, fmax=16000)).float().to(dev)
    window = torch.hann_window(WIN, device=dev)
    pleaf = dense.to(dev).requires_grad_(True)
    noise = torch.randn(B, T, device=dev)

    def port_step():
        with torch.device(dev):
            sig = tp.superfast_forward(f0, syn.split_views(pleaf, sm), SR, P, WIN, noise=noise)["signal"]
        F.mse_loss(reference_get_mel(sig, basis, window).transpose(1, 2), target).backward()

    def port_prep():
        pleaf.grad = None
    port_ms = timed(port_step, port_prep, flush, max(3, steps // 4), 1)
    del pleaf, noise
    torch.cuda.empty_cache()
    return {"B": B, "n_frames": nF, "seconds": T / SR,
            "mel_forward_ms": mel_ms, "mel_backward_kernel_ms": kern_ms, "mel_backward_kernel_bytes": nbytes,
            "mel_backward_kernel_GBps": nbytes / (kern_ms * 1e-3) / 1e9,
            "ddsp_loss_step_ms": step_ms, "reference_eager_ddsp_loss_step_ms": port_ms,
            "speedup_vs_reference": port_ms / step_ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mel_grad.py needs a CUDA device (no fallback)")
    from ddsp_svc_b200 import _lib
    _lib.lib()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    line = {"metric": "mel_grad_ddsp_loss_step", "card": card(),
            "timing": "median of %d steps after %d warm-up, CUDA events, L2 flushed before each step (untimed); "
                      "step = superfast frame scan + synthesis + mel + MSE + autograd backward through both; "
                      "reference = oracle.torch_port.superfast_forward + oracle.mel's operators under autograd, eager, "
                      "same GPU" % (args.steps, args.warmup),
            "shapes": {label: run_shape(B, nF, flush, args.steps, args.warmup) for label, B, nF in SHAPES}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
