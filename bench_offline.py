"""Whole-file conversion time of main.py's loop: 60 s of 44.1 kHz synthetic speech with pauses, converted by a
CombSubSuperFast model with the NSF-HiFiGAN enhancer (key 0, adaptive key 0; synthetic seeded checkpoints of
bench_realtime.write_synthetic, written to a temporary directory).

Two arms on the same modules and the same split, alternated, each timed from the call to the end of a device
synchronise; medians over --steps calls after --warmup calls of each:
  offline   OfflineVC.convert with the segments given: every segment queued on the device, assembled there
  loop      main.py's loop (tests/offline_oracle.main_loop): a host round trip per segment, np.append and the float64
            cross_fade
Prints one JSON line with the card's name and power limit."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

PIECES = [("v", 7.0), ("s", 0.8), ("v", 9.0), ("s", 2.0), ("v", 6.5), ("s", 0.4), ("v", 8.0), ("s", 6.0), ("v", 7.5),
          ("s", 1.2), ("v", 11.6)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_offline.py needs a CUDA device"
    from bench_realtime import write_synthetic
    from ddsp_svc_b200.offline import OfflineVC
    from tests import offline_oracle as oo
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    sr = 44100
    audio = oo.speech(PIECES, sr, seed=60)
    assert audio.shape[0] == 60 * sr
    with tempfile.TemporaryDirectory() as d, contextlib.redirect_stdout(io.StringIO()):
        model_path, rmvpe_path = write_synthetic(d, "CombSubSuperFast")
        vc = OfflineVC(model_path, device="cuda:0", rmvpe_ckpt=rmvpe_path)
        x = torch.from_numpy(audio).to("cuda:0")
        segments = vc.split(x, sr)
        arms = {"offline": lambda: vc.convert(x, sr, segments=segments),
                "loop": lambda: oo.main_loop(vc, audio, sr, segments)}
        times = {k: [] for k in arms}
        for i in range(a.warmup + a.steps):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                if i >= a.warmup:
                    times[name].append(1e3 * (time.perf_counter() - t0))
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({"metric": "whole-file conversion time (ms)", "gpu": q[0] if q else torch.cuda.get_device_name(),
                      "audio": "60 s at 44.1 kHz, %d segments" % len(segments),
                      "model": "CombSubSuperFast + NSF-HiFiGAN enhancer (synthetic weights)",
                      "median_ms": med, "all_ms": times, "speedup": med["loop"] / med["offline"]}))


if __name__ == "__main__":
    main()
