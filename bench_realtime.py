"""Per-block latency of gui.py's real-time callback at the GUI defaults (44.1 kHz, block 0.3 s, crossfade 0.04 s,
extra 2.0 s, enhancer on, key 0), with synthetic checkpoints of a Sins and a CombSubSuperFast model (HuBERT-soft units,
RMVPE, NSF-HiFiGAN enhancer, all seeded; written to a temporary directory).

Three arms, each timed from the call to the end of the block's output copy, median and p99 over --blocks blocks after
--warmup blocks:
  graph    RealtimeVC(graph=True): graphs A and B replayed
  eager    RealtimeVC(graph=False): the same code launched eagerly
  gui      gui.py's own order on the package's modules, with host numpy (F0_Extractor's interpolation, the volume mask)
           and eager torch (SOLA by conv1d, the crossfade) in between: what a patched reference runs
           (conversion_fixtures.GuiBlock)
Prints one JSON line with the card's name and power limit."""
import argparse
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

# HIFIGAN is not used here: it stays importable from this script, with the writer it configures
from conversion_fixtures import HIFIGAN, MODELS, GuiBlock, write_synthetic  # noqa: E402,F401


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_realtime.py needs a CUDA device"
    from ddsp_svc_b200.realtime import RealtimeVC
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    result = {"metric": "realtime block latency (ms)", "gpu": q[0] if q else torch.cuda.get_device_name(),
              "settings": "44.1 kHz, block 0.3 s, crossfade 0.04 s, extra 2.0 s, enhancer key 0", "models": {}}
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as d:
        for name in MODELS:
            sub = os.path.join(d, name)
            os.makedirs(sub)
            model_path, rmvpe_path = write_synthetic(sub, name)
            arms = {}
            for arm in ("graph", "eager", "gui"):
                s = RealtimeVC(model_path, graph=arm == "graph", rmvpe_ckpt=rmvpe_path, device="cuda:0")
                call = s.process if arm != "gui" else GuiBlock(s)
                times = []
                for i in range(a.warmup + a.blocks):
                    x = (0.1 * rng.standard_normal((s.block, 2))).astype(np.float32)
                    t0 = time.perf_counter()
                    call(x)
                    torch.cuda.synchronize()
                    if i >= a.warmup:
                        times.append(1e3 * (time.perf_counter() - t0))
                arms[arm] = {"median_ms": float(np.median(times)), "p99_ms": float(np.percentile(times, 99))}
            result["models"][name] = arms
    print(json.dumps(result))


if __name__ == "__main__":
    main()
