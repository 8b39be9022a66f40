"""Whole-file conversion time of main_diff.py's loop and batch_infer.py's infer(): 60 s of 44.1 kHz synthetic speech
with pauses, converted by a 'DiffusionNew' model at configs/diffusion-new.yaml's sizes (CombSubFast and WaveNet(128, 20,
512, 256), its built-in DDSP model; ContentVec units at layer 12, RMVPE, NSF-HiFiGAN) with DPM-Solver at speedup 10 and
k_step 100 (key 0, formant key 0; synthetic seeded checkpoints of conversion_fixtures.write_synthetic_diff,
written to a temporary directory).

Four arms on the same modules, alternated, each timed from the call to the end of a device synchronise; medians over
--steps calls after --warmup calls of each:
  offline   OfflineDiffVC.convert with the segments given: every segment queued on the device, assembled there
  loop      main_diff.py's loop (tests/offline_diff_oracle.main_diff_loop): a host round trip per segment, np.append
            and the float64 cross_fade
  whole     OfflineDiffVC.convert_whole: the whole file in one model call
  infer     batch_infer.py's infer() (tests/offline_diff_oracle.batch_infer), its output copied to the host
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

from bench_offline import PIECES  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_offline_diff.py needs a CUDA device"
    from conversion_fixtures import write_synthetic_diff
    from ddsp_svc_b200.offline import OfflineDiffVC
    from tests import offline_diff_oracle as odo
    from tests import offline_oracle as oo
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    sr = 44100
    audio = oo.speech(PIECES, sr, seed=60)
    assert audio.shape[0] == 60 * sr
    kw = dict(speedup=10, method="dpm-solver", k_step=100)
    with tempfile.TemporaryDirectory() as d, contextlib.redirect_stdout(io.StringIO()):
        _, diff_path, rmvpe_path = write_synthetic_diff(d, "DiffusionNew")
        vc = OfflineDiffVC(diff_path, device="cuda:0", rmvpe_ckpt=rmvpe_path)
        x = torch.from_numpy(audio).to("cuda:0")
        segments = vc.split(x, sr)
        sliced, whole = vc.settings(**kw), vc.settings(**kw, whole=True)
        arms = {"offline": lambda: vc.convert(x, sr, segments=segments, **kw),
                "loop": lambda: odo.main_diff_loop(vc, audio, sr, segments, sliced),
                "whole": lambda: vc.convert_whole(x, sr, **kw),
                "infer": lambda: odo.batch_infer(vc, audio, sr, whole)}
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
    print(json.dumps({"metric": "whole-file diffusion conversion time (ms)",
                      "gpu": q[0] if q else torch.cuda.get_device_name(),
                      "audio": "60 s at 44.1 kHz, %d segments" % len(segments),
                      "model": "DiffusionNew, WaveNet(128, 20, 512, 256), built-in CombSubFast, dpm-solver, "
                               "speedup 10, k_step 100 (synthetic weights)",
                      "median_ms": med, "all_ms": times, "speedup_sliced": med["loop"] / med["offline"],
                      "speedup_whole": med["infer"] / med["whole"]}))


if __name__ == "__main__":
    main()
