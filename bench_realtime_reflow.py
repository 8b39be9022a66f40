"""Per-block latency of gui_reflow.py's real-time callback at the GUI defaults (44.1 kHz, block 0.5 s, crossfade 0.04 s,
extra 2.0 s, t_start 0.7), with synthetic seeded checkpoints at configs/reflow.yaml's widths (a Unit2Wav with the
velocity network at n_chans 512 x 6 layers, ContentVec units at layer 12, RMVPE, NSF-HiFiGAN; written to a temporary
directory).  Two samplers: 20 Euler steps (reflow.yaml's infer_step) and 5 RK4 steps.

Three arms per sampler, each timed from the call to the end of the block's output copy, median and p99 over --blocks
blocks after --warmup blocks:
  graph    RealtimeReflowVC(graph=True): the block's one graph replayed
  eager    RealtimeReflowVC(graph=False): the same code launched eagerly
  gui      gui_reflow.py's own order on the package's modules, with host numpy (F0_Extractor's interpolation, the volume
           mask) and eager torch (the mask multiply, SOLA by conv1d, the crossfade) in between: what a patched reference
           runs (GuiReflowBlock)
and the eager session's stages from CUDA events on its stream (median ms): RMVPE, units, ddsp, mel, sampler, vocoder and
the tail (mask, resampling, SOLA, crossfade, output copy).  Prints one JSON line with the card's name and power limit."""
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

from conversion_fixtures import GuiReflowBlock, write_synthetic_reflow  # noqa: E402

STAGES = ("rmvpe", "units", "ddsp", "mel", "sampler", "vocoder", "tail")
SAMPLERS = {"euler20": dict(sampling_method="euler", infer_step=20), "rk4_5": dict(sampling_method="rk4", infer_step=5)}


def stage_times(s, xs):
    """the eager session's block split at its stages by CUDA events on its stream -> {stage: [ms per block]}"""
    from ddsp_svc_b200 import frontend, ops
    times = {k: [] for k in STAGES}
    m = s.model
    for x in xs:
        s.upload(x)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]
        with torch.cuda.stream(s.stream), torch.no_grad():
            ev[0].record()
            s.ring.copy_(torch.cat([s.ring[s.block:], s.new_block]))
            audio = s.ring[None]
            f0_10ms = s.rmvpe.infer_batch(audio[:, s.trim:], s.sr)[0]
            f0 = ops.rt_f0_regrid(f0_10ms.contiguous(), 0.01, s.n_frames, s.hop / s.sr, rmvpe=True,
                                  pad=s.start_frame, f0_min=s.f0_min, post_scale=s.pitch_factor)[None, :, None]
            ev[1].record()
            volume = frontend.volume_extract(audio, s.hop)
            mask = frontend.volume_mask(volume, s.threhold)
            units = s.units_encoder.encode(audio, s.sr, s.hop)
            ev[2].record()
            s._draw_noise()
            wav, _, _ = m.ddsp_model(units, f0, volume[..., None], spk_id=s.spk_id, spk_mix_dict=s.spk_mix_dict,
                                     aug_shift=s.aug_shift, noise=s.noise)
            ev[3].record()
            mel = s.vocoder.extract(wav[:, m.start_frame(s.silence_front) * m.block_size:])
            ev[4].record()
            if s.t_start < 1.0:
                mel = m.reflow_model(mel, gt_spec=mel, infer_step=s.infer_step, method=s.method, t_start=s.t_start,
                                     noise=s.reflow_noise)
            ev[5].record()
            out = s.vocoder.infer(mel, f0[:, -mel.shape[1]:], rand_ini=s.gen_rand_ini, noise=s.gen_noise)
            ev[6].record()
            out = frontend.mask_apply_(out.reshape(1, -1).contiguous(), mask, s.block_size, s.mask_offset)
            s._tail(out, s.model_sr)
            ev[7].record()
        s.stream.synchronize()
        for i, k in enumerate(STAGES):
            times[k].append(ev[i].elapsed_time(ev[i + 1]))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_realtime_reflow.py needs a CUDA device"
    from ddsp_svc_b200.realtime import RealtimeReflowVC
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    result = {"metric": "realtime reflow block latency (ms)", "gpu": q[0] if q else torch.cuda.get_device_name(),
              "settings": "44.1 kHz, block 0.5 s, crossfade 0.04 s, extra 2.0 s, t_start 0.7, n_chans 512 x 6 layers, "
                          "contentvec768l12", "samplers": {}}
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as d:
        model_path, rmvpe_path = write_synthetic_reflow(d)
        for name, kw in SAMPLERS.items():
            arms = {}
            for arm in ("graph", "eager", "gui"):
                s = RealtimeReflowVC(model_path, graph=arm == "graph", rmvpe_ckpt=rmvpe_path, device="cuda:0",
                                     t_start=0.7, **kw)
                call = s.process if arm != "gui" else GuiReflowBlock(s)
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
                    xs = [(0.1 * rng.standard_normal((s.block, 2))).astype(np.float32)
                          for _ in range(a.warmup + a.blocks)]
                    st = stage_times(s, xs)
                    arms["eager_stages_ms"] = {k: float(np.median(v[a.warmup:])) for k, v in st.items()}
                del s
            result["samplers"][name] = arms
    print(json.dumps(result))


if __name__ == "__main__":
    main()
