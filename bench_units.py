"""Time the units encoder in its default configuration (contentvec768l12: the fairseq HuBERT-base layout read at layer
12): the kernels (ddsp_svc_b200.Units_Encoder) against the plain-torch oracle run eagerly in fp32 on the same GPU under
torch's defaults (fp32 cuBLAS Linear, cuDNN TF32 convolutions: what the reference runs).  Seeded weights
(tests/units_oracle.seeded_state_dict) and seeded 44.1 kHz audio, hop 512.  For each shape it times the whole encode
(resample, encoder, alignment) and the encoder alone, after a warm-up, flushing L2 before every call and alternating the
arms; medians.  Both arms build their resample taps once per rate outside the timed calls, as the reference caches its
Resample.  Accuracy: relative RMS of the aligned units against float64.  GFLOP counted from the shapes.  Prints one JSON
line per shape with the card and its power limit; --profile instead prints a torch.profiler table of the kernels'
CUDA time per kernel name for one shape.  Writes nothing but a temporary checkpoint in a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from ddsp_svc_b200 import hubert as H  # noqa: E402
from tests import rmvpe_oracle as ro  # noqa: E402
from tests import units_oracle as U  # noqa: E402

SR, HOP, KIND = 44100, 512, "contentvec768l12"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception as e:                                   # noqa: BLE001
        return [torch.cuda.get_device_name(), "unknown (%s)" % e]


def timed(fn, flush):
    flush.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def gflop(B, n16, layers=12):
    """multiply-adds x 2 of the encoder from the shapes: feature convolutions, feature projection, positional
    convolution, the transformer layers (projections, FFN, attention)"""
    L = H.feature_lengths(n16)
    T = L[-1]
    f = 2 * L[0] * 512 * 10 + sum(2 * L[i] * 512 * 512 * k for i, k in zip(range(1, 7), (3, 3, 3, 3, 2, 2)))
    f += 2 * T * 512 * 768 + 2 * T * 768 * 48 * 128
    f += layers * (2 * T * 768 * (3 * 768 + 768 + 2 * 3072) + 4 * T * T * 768)
    return B * f / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--shapes", default="1x2,1x10,1x60,16x10", help="B x seconds, comma separated")
    ap.add_argument("--profile", action="store_true", help="profile the kernels' encode of the first shape instead")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_units.py needs a CUDA device"
    dev = torch.device("cuda")
    name, power = card()
    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, "contentvec.pt")
    _, fsd = U.fairseq_state_dict(0)
    U.save_fairseq(path, fsd, args=U.fairseq_args())
    enc = H.Units_Encoder(KIND, path, device=dev)
    os.remove(path)
    os.rmdir(tmp)
    sd = {k: v.to(dev) for k, v in enc.model.state_dict().items()}
    n_layers, proj, _ = H.KINDS[KIND]
    tabs32 = ro.tables(SR, torch.float32, dev)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device=dev)
    with torch.no_grad():
        for shape in args.shapes.split(","):
            B, secs = (int(v) for v in shape.split("x"))
            g = torch.Generator().manual_seed(B * 100 + secs)
            n = SR * secs
            t = torch.arange(n, dtype=torch.float64) / SR
            f = 110 * 2 ** (torch.rand(B, 1, generator=g, dtype=torch.float64) * 3)
            audio = (0.3 * torch.sin(2 * torch.pi * f * t * (1 + 0.05 * torch.sin(2 * torch.pi * t)))
                     + 0.01 * torch.randn(B, n, generator=g, dtype=torch.float64)).float().to(dev)
            res16 = ro.resample(audio, SR, torch.float32, tabs32).contiguous()
            if args.profile:
                enc.encode_batch(audio, SR, HOP)
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    enc.encode_batch(audio, SR, HOP)
                    torch.cuda.synchronize()
                print("profile %s (%s, %s)" % (shape, name, power))
                print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
                return

            def eager(whole):
                torch.backends.cuda.matmul.allow_tf32 = False            # torch's defaults
                torch.backends.cudnn.allow_tf32 = True
                if whole:
                    return U.units_encode(KIND, sd, audio, SR, HOP, torch.float32, batch=B > 1, tabs=tabs32)
                return U.encode(sd, res16, n_layers, proj, 0, torch.float32)

            arms = {"kernels": (lambda: enc.encode_batch(audio, SR, HOP),
                                lambda: enc.model._run(res16, 0, n_layers, proj)),
                    "eager_fp32": (lambda: eager(True), lambda: eager(False))}
            for w, net in arms.values():                               # warm-up
                w()
                net()
            torch.cuda.synchronize()
            times = {k: ([], []) for k in arms}
            for _ in range(args.reps):
                for k, (w, net) in arms.items():
                    times[k][0].append(timed(w, flush))
                    times[k][1].append(timed(net, flush))
            want = U.units_encode(KIND, sd, audio.double(), SR, HOP, torch.float64, batch=B > 1)
            scale = want.norm().item()
            acc = {k: ((w().double() - want).norm().item() / scale) for k, (w, _) in arms.items()}
            res = dict(shape="%dx%ds@%d" % (B, secs, SR), frames=int(want.shape[1]), card=name, power_limit=power,
                       gflop=round(gflop(B, res16.shape[1]), 2),
                       whole_ms={k: median(v[0]) for k, v in times.items()},
                       encoder_ms={k: median(v[1]) for k, v in times.items()}, units_rel_rms=acc)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
