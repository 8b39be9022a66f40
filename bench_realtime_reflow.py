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
import yaml

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_realtime import HIFIGAN, GuiBlock  # noqa: E402

STAGES = ("rmvpe", "units", "ddsp", "mel", "sampler", "vocoder", "tail")
SAMPLERS = {"euler20": dict(sampling_method="euler", infer_step=20), "rk4_5": dict(sampling_method="rk4", infer_step=5)}


def write_front(d, encoder="contentvec768l12"):
    """seeded checkpoints of what every diffusion / reflow session loads besides its model, in directory d: the units
    encoder, RMVPE and NSF-HiFiGAN (voc/model.ckpt) -> the config's data and vocoder sections"""
    import ddsp_svc_b200 as pkg
    from ddsp_svc_b200 import dropin
    from ddsp_svc_b200.hifigan import Generator
    os.makedirs(os.path.join(d, "voc"), exist_ok=True)
    if encoder == "hubertsoft":
        enc_path, n_unit = os.path.join(d, "hubert.pt"), 256
        torch.save(pkg.HubertSoft().state_dict(), enc_path)
    else:
        from tests import units_oracle
        enc_path, n_unit = os.path.join(d, "contentvec.pt"), 768
        units_oracle.save_fairseq(enc_path, units_oracle.fairseq_state_dict(0)[1], args=units_oracle.fairseq_args())
    torch.save({"model": pkg.E2E0(4, 1, (2, 2)).state_dict()}, os.path.join(d, "rmvpe.pt"))
    with open(os.path.join(d, "voc", "config.json"), "w") as f:
        json.dump(HIFIGAN, f)
    gen = Generator(dropin.DotDict(HIFIGAN))
    torch.save({"generator": gen.state_dict()}, os.path.join(d, "voc", "model.ckpt"))
    return ({"sampling_rate": 44100, "block_size": 512, "encoder": encoder, "encoder_ckpt": enc_path,
             "encoder_sample_rate": 16000, "encoder_hop_size": 320, "encoder_out_channels": n_unit},
            {"type": "nsf-hifigan", "ckpt": os.path.join(d, "voc", "model.ckpt")})


def write_synthetic_reflow(d, n_chans=512, n_layers=6, encoder="contentvec768l12", n_spk=2, model_type="RectifiedFlow"):
    """seeded checkpoints of a reflow session in directory d -> (model path, rmvpe path).  The velocity network's
    parameters are all non-zero (tests/reflow_oracle.seeded_weights; the default init zeroes its output projection);
    ``encoder``: 'contentvec768l12' (reflow.yaml) or 'hubertsoft'"""
    import ddsp_svc_b200 as pkg
    from tests import reflow_oracle
    torch.manual_seed(0)
    data, voc = write_front(d, encoder)
    n_unit = data["encoder_out_channels"]
    cfg = {"data": data,
           "model": {"type": model_type, "win_length": 2048, "n_layers": n_layers, "n_chans": n_chans,
                     "use_pitch_aug": True, "n_spk": n_spk},
           "vocoder": voc}
    with open(os.path.join(d, "config.yaml"), "w") as f:
        yaml.safe_dump(cfg, f)
    model = pkg.Unit2Wav(44100, 512, 2048, n_unit, n_spk, True, HIFIGAN["num_mels"], n_layers, n_chans)
    reflow_oracle.seeded_weights(model.reflow_model.velocity_fn, 7)
    torch.save({"model": model.state_dict()}, os.path.join(d, "model.pt"))
    return os.path.join(d, "model.pt"), os.path.join(d, "rmvpe.pt")


class GuiReflowBlock(GuiBlock):
    """gui_reflow.py's audio_callback and SvcDDSP.infer in their own order on a RealtimeReflowVC's modules and draws
    (the session's static buffers, which hold its last draws), with host numpy and eager torch in between.  The speaker
    mix is the session's (gated on use_spk_mix, where gui_reflow.py:137 passes spk_mix_dict regardless)."""

    def __call__(self, indata):
        s = self.s
        f0, volume, mask, units = self.front(indata)
        formant_shift_key = torch.from_numpy(np.array([[float(s.formant_shift_key)]])).float().to(s.device)
        with torch.no_grad():
            output = s.model(units, f0, volume[..., None], spk_id=s.spk_id, spk_mix_dict=s.spk_mix_dict,
                             aug_shift=formant_shift_key, vocoder=s.vocoder, infer=True, return_wav=True,
                             infer_step=s.infer_step, method=s.method, t_start=s.t_start,
                             silence_front=s.silence_front, use_tqdm=False, ddsp_noise=s.noise,
                             reflow_noise=s.reflow_noise, rand_ini=s.gen_rand_ini, sine_noise=s.gen_noise)
            output *= mask[:, -output.shape[-1]:]
        return self.tail(output, s.model_sr)


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
