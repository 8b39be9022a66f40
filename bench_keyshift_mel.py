"""The key-shifted mel of preprocess.py's pitch augmentation (STFT.get_mel(audio, keyshift), keyshift ~ U(-5, 5)) on the
kernel (mel.STFT.get_mel_keyshift: one launch of mel_keyshift_kernel) against the reference's algorithm run eagerly in
fp32 on the same GPU (pad, torch.stft on cuFFT, magnitude, scaling, matmul, log; tests/keyshift_mel_oracle.get_mel with
its tables on the device).  Prints one JSON line.

    python bench_keyshift_mel.py [--steps 20] [--warmup 3]

Shapes: preprocess.py's call, 1 x 10 s with a keyshift drawn from a seeded U(-5, 5) per call (every drawn length's
table built before timing; the first use of a length builds its table, timed separately as table_build_ms), and a batch
of 16 x 10 s at keyshift -5 (n' = 1534) and +4.98 (n' = 2731, prime).  Each call is timed with CUDA events after the L2
was flushed (256 MiB memset, untimed); medians are reported.  Accuracy: max and RMS log-mel error of both sides against
float64 on the first row.  Needs a CUDA device; there is no fallback."""
import argparse
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_superfast_grad import card, timed  # noqa: E402

SR, HOP, T10 = 44100, 512, 441000


def errors(out, ref):
    d = out[:1].double().cpu() - ref
    return {"max": d.abs().max().item(), "rms": d.pow(2).mean().sqrt().item()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_keyshift_mel.py needs a CUDA device (no fallback)")
    from ddsp_svc_b200 import mel as pm
    from tests import keyshift_mel_oracle as ko
    dev = torch.device("cuda", torch.cuda.current_device())
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)      # > 50 MB L2
    st = pm.STFT(SR, 128, 2048, 2048, HOP, 40, 16000)
    basis = ko.basis(device=dev)
    windows = {}

    def reference(y, keyshift):
        n = ko.n_fft_new(keyshift)
        if n not in windows:
            windows[n] = torch.hann_window(n, device=dev)
        with torch.no_grad():
            return ko.get_mel(y, HOP, keyshift, basis, windows[n])

    g = torch.Generator().manual_seed(31)
    shapes = {}

    # preprocess.py: one clip per call, a fresh keyshift per call
    rng = random.Random(5)
    shifts = [rng.uniform(-5, 5) for _ in range(args.steps + args.warmup)]
    y1 = (0.1 * torch.randn(1, T10, generator=g)).to(dev)
    t0 = time.perf_counter()
    pm._keyshift_tables.get(pm.keyshift_n_fft(2048, 4.321), dev)                # one table, host float64 + upload
    build_ms = 1e3 * (time.perf_counter() - t0)
    for k in shifts:
        st.get_mel_keyshift(y1, k)
        reference(y1, k)
    it = iter(range(len(shifts)))
    kern_ms = timed(lambda: st.get_mel_keyshift(y1, shifts[next(it) % len(shifts)]), lambda: None, flush, args.steps,
                    args.warmup)
    it = iter(range(len(shifts)))
    ref_ms = timed(lambda: reference(y1, shifts[next(it) % len(shifts)]), lambda: None, flush, args.steps, args.warmup)
    want = ko.mel64(y1[:1].cpu(), HOP, shifts[0])
    shapes["preprocess_b1_10s_uniform5"] = {
        "B": 1, "seconds": T10 / SR, "kernel_ms": kern_ms, "reference_eager_ms": ref_ms, "speedup": ref_ms / kern_ms,
        "table_build_ms": build_ms, "keyshift_error_row": shifts[0],
        "kernel_vs_float64": errors(st.get_mel_keyshift(y1, shifts[0]), want),
        "reference_vs_float64": errors(reference(y1, shifts[0]), want)}

    # a batch at both ends of preprocess's range
    yb = (0.1 * torch.randn(16, T10, generator=g)).to(dev)
    for k in (-5.0, 4.98):
        kern_ms = timed(lambda: st.get_mel_keyshift(yb, k), lambda: None, flush, args.steps, args.warmup)
        ref_ms = timed(lambda: reference(yb, k), lambda: None, flush, args.steps, args.warmup)
        want = ko.mel64(yb[:1].cpu(), HOP, k)
        shapes["batch_b16_10s_ks%+g" % k] = {
            "B": 16, "seconds": T10 / SR, "n_fft": pm.keyshift_n_fft(2048, k), "kernel_ms": kern_ms,
            "reference_eager_ms": ref_ms, "speedup": ref_ms / kern_ms,
            "kernel_vs_float64": errors(st.get_mel_keyshift(yb, k), want),
            "reference_vs_float64": errors(reference(yb, k), want)}
    line = {"metric": "keyshift_mel", "card": card(),
            "timing": "median of %d calls after %d warm-up, CUDA events, L2 flushed before each call (untimed); "
                      "reference = the reference's get_mel algorithm eager in fp32 on the same GPU (torch.stft / cuFFT)"
                      % (args.steps, args.warmup),
            "shapes": shapes}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
