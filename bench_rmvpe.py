"""Time the RMVPE pitch extractor: the kernels (ddsp_svc_b200.RMVPE.infer_batch) against the plain-torch oracle run
eagerly on the same GPU, under torch's defaults (cuDNN TF32, what the reference runs) and with TF32 off.  Seeded
weights with calibrated BatchNorm (tests/rmvpe_oracle.seeded_model) and seeded 44.1 kHz audio.  For each shape it times
the whole path (resample, log-mel, network, decode) and the network alone, after a warm-up, flushing L2 before every
call and alternating the arms; medians.  Every arm builds its host tables (resample taps, window, mel basis) once per
rate outside the timed calls, as the reference caches them.  Accuracy: salience relative RMS against float64 and the number of decoded
frames whose f0 differs from float64's by more than 1e-4 relative.  Prints one JSON line per shape with the card and
its power limit.  Writes nothing but a temporary checkpoint in a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from ddsp_svc_b200 import rmvpe as R  # noqa: E402
from tests import rmvpe_oracle as ro  # noqa: E402

SR = 44100


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception as e:                                   # noqa: BLE001
        return [torch.cuda.get_device_name(), "unknown (%s)" % e]


def timed(fn, flush, reps):
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--shapes", default="1x2,1x10,16x10", help="B x seconds, comma separated")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rmvpe.py needs a CUDA device"
    dev = torch.device("cuda")
    name, power = card()
    with torch.no_grad():
        model = ro.seeded_model().to(dev)
        tmp = tempfile.mkdtemp()
        path = os.path.join(tmp, "model.pt")
        torch.save({"model": model.state_dict()}, path)
        ex = R.RMVPE(path)
        os.remove(path)
        os.rmdir(tmp)
        flush = torch.empty(64 << 20, dtype=torch.uint8, device=dev)
        for shape in args.shapes.split(","):
            B, secs = (int(v) for v in shape.split("x"))
            g = torch.Generator().manual_seed(B * 100 + secs)
            n = SR * secs
            t = torch.arange(n, dtype=torch.float64) / SR
            f = 110 * 2 ** (torch.rand(B, 1, generator=g, dtype=torch.float64) * 3)
            audio64 = (0.3 * torch.sin(2 * torch.pi * f * t * (1 + 0.05 * torch.sin(2 * torch.pi * t)))
                       + 0.01 * torch.randn(B, n, generator=g, dtype=torch.float64)).to(dev)
            audio = audio64.float()
            ref_f0, ref_sal = ro.infer(model, audio64, SR)
            tabs32 = ro.tables(SR, torch.float32, dev)      # built once per rate, outside the timed calls
            mel32 = ro.log_mel(ro.resample(audio, SR, torch.float32, tabs32), dtype=torch.float32, tabs=tabs32)
            nf = mel32.shape[-1]
            mel_pad = torch.nn.functional.pad(mel32, (0, 32 * ((nf - 1) // 32 + 1) - nf))

            def eager(tf32, whole):
                torch.backends.cuda.matmul.allow_tf32 = tf32
                torch.backends.cudnn.allow_tf32 = tf32
                if whole:
                    return ro.infer(model, audio, SR, dtype=torch.float32, tabs=tabs32)
                return ro.salience(model, mel_pad, torch.float32)

            arms = {
                "kernels": (lambda: ex.infer_batch(audio, SR), lambda: ex.model._salience(mel_pad.transpose(1, 2)
                                                                                              .unsqueeze(-1))),
                "eager_tf32": (lambda: eager(True, True), lambda: eager(True, False)),
                "eager_fp32": (lambda: eager(False, True), lambda: eager(False, False)),
            }
            times = {k: ([], []) for k in arms}
            for k, (w, net) in arms.items():                 # warm-up
                w(); net()
            torch.cuda.synchronize()
            for _ in range(args.reps):
                for k, (w, net) in arms.items():
                    times[k][0].extend(timed(w, flush, 1))
                    times[k][1].extend(timed(net, flush, 1))
            acc = {}
            scale = ref_sal.pow(2).mean().sqrt().item()
            sal_k, nfk = ex.salience_batch(audio, SR)
            f0_k = ex.infer_batch(audio, SR)
            for k, (sal, f0) in {"kernels": (sal_k[:, :nfk], f0_k),
                                 "eager_tf32": eager(True, True)[::-1], "eager_fp32": eager(False, True)[::-1]}.items():
                rel = (sal.double() - ref_sal).pow(2).mean().sqrt().item() / scale
                differ = int(((f0.double() - ref_f0).abs() > 1e-4 * ref_f0.abs().clamp(min=1e-30)).sum())
                acc[k] = dict(salience_rel_rms=rel, f0_frames_differ=differ)
            torch.backends.cuda.matmul.allow_tf32 = False
            torch.backends.cudnn.allow_tf32 = True
            res = dict(shape="%dx%ds@%d" % (B, secs, SR), frames=int(ref_f0.shape[1]), card=name, power_limit=power,
                       whole_ms={k: median(v[0]) for k, v in times.items()},
                       network_ms={k: median(v[1]) for k, v in times.items()}, accuracy=acc)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
