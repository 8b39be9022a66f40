"""Per-block latency of gui.py's real-time callback at the GUI defaults (44.1 kHz, block 0.3 s, crossfade 0.04 s,
extra 2.0 s, enhancer on, key 0), with synthetic checkpoints of a Sins and a CombSubSuperFast model (HuBERT-soft units,
RMVPE, NSF-HiFiGAN enhancer, all seeded; written to a temporary directory).

Three arms, each timed from the call to the end of the block's output copy, median and p99 over --blocks blocks after
--warmup blocks:
  graph    RealtimeVC(graph=True): graphs A and B replayed
  eager    RealtimeVC(graph=False): the same code launched eagerly
  gui      gui.py's own order on the package's modules, with host numpy (F0_Extractor's interpolation, the volume mask)
           and eager torch (SOLA by conv1d, the crossfade) in between: what a patched reference runs (gui_block)
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
import torch.nn.functional as F
import yaml

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

MODELS = {"Sins": {"type": "Sins", "n_harmonics": 128, "n_mag_allpass": 256, "n_mag_noise": 256, "n_spk": 2},
          "CombSubSuperFast": {"type": "CombSubSuperFast", "win_length": 2048, "n_spk": 2}}
HIFIGAN = dict(resblock="1", num_mels=128, sampling_rate=44100, upsample_rates=[8, 8, 8],
               upsample_kernel_sizes=[16, 16, 16], upsample_initial_channel=128, resblock_kernel_sizes=[3, 7, 11],
               resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], n_fft=2048, win_size=2048, hop_size=512,
               fmin=40, fmax=16000)


def write_synthetic(d, model_type):
    """seeded checkpoints of the whole session in directory d -> (model path, rmvpe path)"""
    import ddsp_svc_b200 as pkg
    from ddsp_svc_b200 import dropin
    from ddsp_svc_b200.hifigan import Generator
    torch.manual_seed(0)
    os.makedirs(os.path.join(d, "enh"), exist_ok=True)
    torch.save(pkg.HubertSoft().state_dict(), os.path.join(d, "hubert.pt"))
    torch.save({"model": pkg.E2E0(4, 1, (2, 2)).state_dict()}, os.path.join(d, "rmvpe.pt"))
    with open(os.path.join(d, "enh", "config.json"), "w") as f:
        json.dump(HIFIGAN, f)
    gen = Generator(dropin.DotDict(HIFIGAN))
    torch.save({"generator": gen.state_dict()}, os.path.join(d, "enh", "model.ckpt"))
    cfg = {"data": {"sampling_rate": 44100, "block_size": 512, "encoder": "hubertsoft",
                    "encoder_ckpt": os.path.join(d, "hubert.pt"), "encoder_sample_rate": 16000,
                    "encoder_hop_size": 320, "encoder_out_channels": 256},
           "model": MODELS[model_type], "enhancer": {"type": "nsf-hifigan", "ckpt": os.path.join(d, "enh", "model.ckpt")}}
    with open(os.path.join(d, "config.yaml"), "w") as f:
        yaml.safe_dump(cfg, f)
    model = dropin.build_model(dropin.DotDict(cfg))
    torch.save({"model": model.state_dict()}, os.path.join(d, "model.pt"))
    return os.path.join(d, "model.pt"), os.path.join(d, "rmvpe.pt")


def phase_vocoder(a, b, fade_out, fade_in):
    """gui.py's phase_vocoder in eager torch"""
    window = torch.sqrt(fade_out * fade_in)
    fa, fb = torch.fft.rfft(a * window), torch.fft.rfft(b * window)
    absab = torch.abs(fa) + torch.abs(fb)
    n = a.shape[0]
    absab[1:(n - 1) // 2 + 1] *= 2
    pa = torch.angle(fa)
    d = torch.angle(fb) - pa
    d = d - 2 * np.pi * torch.floor(d / 2 / np.pi + 0.5)
    w = 2 * np.pi * torch.arange(n // 2 + 1).to(a) + d
    t = torch.arange(n).unsqueeze(-1).to(a) / n
    return a * fade_out ** 2 + b * fade_in ** 2 + torch.sum(absab * torch.cos(w * t + pa), -1) * window / n


class GuiBlock:
    """gui.py's audio_callback and SvcDDSP.infer in their own order on a session's modules (its models, tables and
    noise buffers, which hold the session's last draws), with host numpy and eager torch in between.  phase_vocoder
    runs in float64, where torch's fp32 phase w t would be off by up to 3e-4 rad."""

    def __init__(self, s):
        from tests import realtime_oracle as ro   # the float64 statement of F0_Extractor's interpolation
        self.s, self.ro = s, ro
        self.input_wav = np.zeros(s.n_in, dtype=np.float32)
        self.sola_buffer = torch.zeros(s.cf, device=s.device)

    def __call__(self, indata):
        from ddsp_svc_b200 import frontend
        s, dev = self.s, self.s.device
        self.input_wav[:] = np.roll(self.input_wav, -s.block)
        self.input_wav[-s.block:] = np.asarray(indata, np.float32).mean(axis=1, dtype=np.float32)
        audio_t = torch.from_numpy(self.input_wav).to(dev)[None]
        f0_10 = s.rmvpe.infer_batch(audio_t[:, s.trim:], s.sr)[0].cpu().numpy()
        f0 = self.ro.rmvpe_f0(f0_10, s.hop, s.sr, s.n_frames, s.start_frame, s.f0_min, s.pitch_adjust)
        f0 = torch.from_numpy(f0).to(dev)[None, :, None]
        volume = frontend.volume_extract(audio_t, s.hop)
        mask = (volume[0].cpu().numpy() > np.float32(10 ** (s.threhold / 20))).astype("float")
        mask = np.pad(mask, (4, 4), constant_values=(mask[0], mask[-1]))
        mask = np.array([np.max(mask[n:n + 9]) for n in range(len(mask) - 8)])
        mask = torch.from_numpy(mask).float().to(dev)[None, :, None].permute(0, 2, 1)
        mask = F.interpolate(torch.cat((mask, mask[:, :, -1:]), 2), size=mask.shape[-1] * s.block_size + 1,
                             mode="linear", align_corners=True)[:, :, :-1].permute(0, 2, 1).squeeze(-1)
        units = s.units_encoder.encode(audio_t, s.sr, s.hop)
        with torch.no_grad():
            out, _, _ = s.model(units, f0, volume[..., None], spk_id=s.spk_id, spk_mix_dict=s.spk_mix_dict,
                                noise=s.noise)
            out *= mask
            if s.use_enhancer:
                key = s.key
                if key == "auto":
                    key = max(0, np.ceil(12 * np.log2(float(torch.max(f0[:, s.start_frame:]) / 760))))
                out, _ = s.enhancer.enhance(out, s.model_sr, f0, s.block_size, adaptive_key=key,
                                            silence_front=s.silence_front, rand_ini=s.gen_rand_ini, noise=s.gen_noise)
        audio = out.squeeze()
        if s.out_sr != s.sr:
            audio = s.to_device_rate(audio[None].contiguous(), s.out_sr)[0]
        temp = audio[-s.block - s.cf - s.search - s.delay:-s.delay]
        conv_input = temp[None, None, :s.cf + s.search]
        nom = F.conv1d(conv_input, self.sola_buffer[None, None, :])
        den = torch.sqrt(F.conv1d(conv_input ** 2, torch.ones(1, 1, s.cf, device=dev)) + 1e-8)
        shift = torch.argmax(nom[0, 0] / den[0, 0])
        temp = temp[shift:shift + s.block + s.cf].clone()
        if s.use_pv:
            temp[:s.cf] = phase_vocoder(self.sola_buffer.double(), temp[:s.cf].double(), s.fade_out.double(),
                                           s.fade_in.double()).float()
        else:
            temp[:s.cf] *= s.fade_in
            temp[:s.cf] += self.sola_buffer * s.fade_out
        self.sola_buffer = temp[-s.cf:]
        return temp[:-s.cf, None].repeat(1, 2).cpu().numpy()


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
