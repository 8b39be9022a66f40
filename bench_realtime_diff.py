"""Per-block latency of gui_diff.py's real-time callback at the GUI defaults (44.1 kHz, block 0.5 s, crossfade 0.04 s,
extra 2.0 s, k_step 100, diff_acc 10), with synthetic seeded checkpoints at configs/diffusion-new.yaml's widths (a
'DiffusionNew' Unit2Wav: CombSubFast and WaveNet(128, 20, 512, 256); ContentVec units at layer 12, RMVPE, NSF-HiFiGAN;
written to a temporary directory).  Four settings: DDIM (the GUI's default method), DPM-Solver with diff_silence off and
on, and a 'Diffusion' Unit2Mel (WaveNet(128, 20, 512, 256), configs/diffusion.yaml) paired with a CombSub DDSP model,
DDIM.

Three arms per setting, each timed from the call to the end of the block's output copy, median and p99 over --blocks
blocks after --warmup blocks:
  graph    RealtimeDiffVC(graph=True): the block's one graph replayed
  eager    RealtimeDiffVC(graph=False): the same code launched eagerly
  gui      gui_diff.py's own order on the package's modules, with host numpy (F0_Extractor's interpolation, the volume
           mask) and eager torch (the mask multiply, SOLA by conv1d, the crossfade) in between: what a patched reference
           runs (GuiDiffBlock)
and the eager session's stages from CUDA events on its stream (median ms): front (RMVPE, volume, mask, units), ddsp (the
external DDSP model), diffusion (the model's call: its DDSP, the mel and the sampler), vocoder and the tail (mask,
resampling, SOLA, crossfade, output copy).  Prints one JSON line with the card's name and power limit."""
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

# DDSP_MODELS is not used here: it stays importable from this script, with the writer whose ``ddsp`` keys it holds
from conversion_fixtures import DDSP_MODELS, GuiDiffBlock, write_synthetic_diff  # noqa: E402,F401

SETTINGS = {
    "ddim": dict(model="DiffusionNew", diff_method="ddim"),
    "dpm": dict(model="DiffusionNew", diff_method="dpm-solver"),
    "dpm_silence": dict(model="DiffusionNew", diff_method="dpm-solver", diff_silence=True),
    "unit2mel_combsub_ddim": dict(model="Diffusion", ddsp="CombSub", diff_method="ddim"),
}
STAGES = ("front", "ddsp", "diffusion", "vocoder", "tail")


def stage_times(s, xs):
    """the eager session's blocks split at its stages by CUDA events on its stream -> {stage: [ms per block]}; the
    session's parts are wrapped on the instance for the measurement and restored after"""
    marks = []

    def timed(fn, name):
        def call(*a, **k):
            out = fn(*a, **k)
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(s.stream)
            marks.append((name, ev))
            return out
        return call

    saved = (s.ddsp_model, s.diff.model)
    s._front = timed(s._front, "front")
    if s.ddsp_model is not None:
        s.ddsp_model = timed(s.ddsp_model, "ddsp")
    s.diff.model = timed(s.diff.model, "diffusion")
    s.diff.vocoder.infer = timed(s.diff.vocoder.infer, "vocoder")
    s._tail = timed(s._tail, "tail")
    times = {k: [] for k in STAGES}
    try:
        for x in xs:
            s.upload(x)
            marks.clear()
            start = torch.cuda.Event(enable_timing=True)
            start.record(s.stream)
            s.run()
            s.stream.synchronize()
            prev = start
            for name, ev in marks:
                times[name].append(prev.elapsed_time(ev))
                prev = ev
    finally:
        s.ddsp_model, s.diff.model = saved
        del s._front, s._tail, s.diff.vocoder.infer                     # the classes' methods again
    return {k: v for k, v in times.items() if v}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--settings", default=",".join(SETTINGS), help="comma-separated keys of SETTINGS")
    a = ap.parse_args()
    names = a.settings.split(",")
    for n in names:
        if n not in SETTINGS:
            ap.error("unknown setting %r (one of %s)" % (n, ", ".join(SETTINGS)))
    assert torch.cuda.is_available(), "bench_realtime_diff.py needs a CUDA device"
    from ddsp_svc_b200.realtime import RealtimeDiffVC
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    result = {"metric": "realtime diffusion block latency (ms)", "gpu": q[0] if q else torch.cuda.get_device_name(),
              "settings": "44.1 kHz, block 0.5 s, crossfade 0.04 s, extra 2.0 s, k_step 100, diff_acc 10, "
                          "WaveNet(128, 20, 512, 256), contentvec768l12", "blocks": a.blocks, "runs": {}}
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as d:
        for name in names:
            cfg = dict(SETTINGS[name])
            sub = os.path.join(d, name)
            ddsp_path, diff_path, rmvpe_path = write_synthetic_diff(sub, cfg.pop("model"), ddsp=cfg.pop("ddsp", None))
            arms = {}
            for arm in ("graph", "eager", "gui"):
                s = RealtimeDiffVC(ddsp_path, diff_path, graph=arm == "graph", rmvpe_ckpt=rmvpe_path, device="cuda:0",
                                   k_step=100, diff_acc=10, **cfg)
                call = s.process if arm != "gui" else GuiDiffBlock(s)
                times = []
                for i in range(a.warmup + a.blocks):
                    x = (0.1 * rng.standard_normal((s.block, 2))).astype(np.float32)
                    t0 = time.perf_counter()
                    call(x)
                    torch.cuda.synchronize()
                    if i >= a.warmup:
                        times.append(1e3 * (time.perf_counter() - t0))
                arms[arm] = {"median_ms": float(np.median(times)), "p99_ms": float(np.percentile(times, 99))}
                if arm == "eager":
                    n = min(a.blocks, 50)
                    xs = [(0.1 * rng.standard_normal((s.block, 2))).astype(np.float32) for _ in range(a.warmup + n)]
                    st = stage_times(s, xs)
                    arms["eager_stages_ms"] = {k: float(np.median(v[a.warmup:])) for k, v in st.items()}
                del s
            result["runs"][name] = arms
    print(json.dumps(result))


if __name__ == "__main__":
    main()
