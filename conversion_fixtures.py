"""What the conversion tests and the real-time benchmarks share: seeded synthetic checkpoints of every session type
(``write_synthetic``, ``write_front``, ``write_synthetic_reflow``, ``write_synthetic_diff``), the GUIs' blocks in
their own order on a session's modules (``GuiBlock``, ``GuiReflowBlock``, ``GuiDiffBlock``: what the sessions are
compared against), and the tests' helpers: a converter built with its stdout silenced, the seeded voice fed to a
session block by block, and one session's draws handed to another.

It sits beside the bench scripts rather than in tests/ so that both import it and neither imports the other; it reads
the float64 statements it needs from tests/ (realtime_oracle, reflow_oracle, units_oracle)."""
import contextlib
import io
import json
import os

import numpy as np
import torch
import torch.nn.functional as F
import yaml

MODELS = {"Sins": {"type": "Sins", "n_harmonics": 128, "n_mag_allpass": 256, "n_mag_noise": 256, "n_spk": 2},
          "CombSubSuperFast": {"type": "CombSubSuperFast", "win_length": 2048, "n_spk": 2}}
DDSP_MODELS = dict(MODELS, CombSub={"type": "CombSub", "n_mag_allpass": 256, "n_mag_harmonic": 512,
                                    "n_mag_noise": 256, "n_spk": 2})
HIFIGAN = dict(resblock="1", num_mels=128, sampling_rate=44100, upsample_rates=[8, 8, 8],
               upsample_kernel_sizes=[16, 16, 16], upsample_initial_channel=128, resblock_kernel_sizes=[3, 7, 11],
               resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], n_fft=2048, win_size=2048, hop_size=512,
               fmin=40, fmax=16000)


# ---- seeded checkpoints ---------------------------------------------------------------------------------------------
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


def write_synthetic_diff(d, model_type="DiffusionNew", n_chans=512, n_layers=20, encoder="contentvec768l12", n_spk=2,
                         ddsp=None, k_step_max=100):
    """seeded checkpoints of a diffusion session in directory d -> (DDSP model path or None, diffusion model path, rmvpe
    path).  model_type: 'Diffusion', 'DiffusionNew' or 'DiffusionFast'; the denoiser's parameters are all non-zero
    (tests/reflow_oracle.seeded_weights; the default init zeroes WaveNet's output projection); ``ddsp``: a key of
    DDSP_MODELS for a DDSP checkpoint with the same data section"""
    from ddsp_svc_b200 import diffusion_vocoder, dropin
    from tests import reflow_oracle
    torch.manual_seed(0)
    data, voc = write_front(d, encoder)
    model = {"type": model_type, "n_layers": n_layers, "n_chans": n_chans, "n_hidden": 256, "win_length": 2048,
             "k_step_max": k_step_max, "use_pitch_aug": True, "n_spk": n_spk}
    cfg = dropin.DotDict({"data": data, "model": model, "vocoder": voc})
    os.makedirs(os.path.join(d, "diff"), exist_ok=True)
    with open(os.path.join(d, "diff", "config.yaml"), "w") as f:
        yaml.safe_dump(dict(cfg), f)
    net = diffusion_vocoder.build_model(cfg, HIFIGAN["num_mels"])
    denoiser = (net.decoder if model_type == "Diffusion" else net.diff_model).denoise_fn
    reflow_oracle.seeded_weights(denoiser, 7, gain=0.5)
    torch.save({"model": net.state_dict()}, os.path.join(d, "diff", "model.pt"))
    ddsp_path = None
    if ddsp is not None:
        os.makedirs(os.path.join(d, "ddsp"), exist_ok=True)
        dcfg = {"data": data, "model": DDSP_MODELS[ddsp]}
        with open(os.path.join(d, "ddsp", "config.yaml"), "w") as f:
            yaml.safe_dump(dcfg, f)
        ddsp_path = os.path.join(d, "ddsp", "model.pt")
        torch.save({"model": dropin.build_model(dropin.DotDict(dcfg)).state_dict()}, ddsp_path)
    return ddsp_path, os.path.join(d, "diff", "model.pt"), os.path.join(d, "rmvpe.pt")


# ---- the GUIs' blocks in their own order ----------------------------------------------------------------------------
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

    def front(self, indata):
        """the ring buffer, f0, volume, the upsampled mask and the units of SvcDDSP.infer"""
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
        return f0, volume, mask, units

    def __call__(self, indata):
        s = self.s
        f0, volume, mask, units = self.front(indata)
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
        return self.tail(out, s.out_sr)

    def tail(self, out, out_sr):
        """audio_callback after SvcDDSP.infer: resampling, SOLA by conv1d, the crossfade or phase vocoder"""
        s, dev = self.s, self.s.device
        audio = out.squeeze()
        if out_sr != s.sr:
            audio = s.to_device_rate(audio[None].contiguous(), out_sr)[0]
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


class GuiDiffBlock(GuiBlock):
    """gui_diff.py's audio_callback and SvcDDSP.infer in their own order on a RealtimeDiffVC's modules and draws (the
    session's static buffers, which hold its last draws), with host numpy and eager torch in between"""

    def __call__(self, indata):
        s = self.s
        f0, volume, mask, units = self.front(indata)
        volume = volume[..., None]
        with torch.no_grad():
            if s.ddsp_model is None:
                output = None
            else:
                output, _, _ = s.ddsp_model(units, f0, volume, spk_id=s.spk_id, spk_mix_dict=s.spk_mix_dict,
                                            noise=s.ext_noise)
            output = s.diff.infer(output, f0, units, volume, acc=s.diff_acc, spk_id=s.spk_id, k_step=s.k_step,
                                  method=s.diff_method, silence_front=s.silence_front, use_silence=s.diff_silence,
                                  spk_mix_dict=s.spk_mix_dict, **s.draws())
            output *= mask
        return self.tail(output, s.model_sr)


# ---- test helpers ---------------------------------------------------------------------------------------------------
def quiet(fn, *a, **k):
    """fn(*a, **k) with its stdout (the loaders' and the enhancer's prints) silenced"""
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def build_session(cls, ckpt, **kw):
    """a converter of class ``cls`` on cuda:0 from a writer's paths (the model path(s), then RMVPE's), built quietly"""
    return quiet(cls, *ckpt[:-1], rmvpe_ckpt=ckpt[-1], device="cuda:0", **kw)


def blocks(s, seed=0, quiet_stretch=False, n_blocks=5):
    """n_blocks stereo blocks [block, 2] for session s: a seeded voice with vibrato; with ``quiet_stretch``, part of
    the first block is 80 dB down so that the mask closes"""
    rng = np.random.default_rng(seed)
    t = np.arange(n_blocks * s.block) / s.sr
    x = 0.3 * np.sin(2 * np.pi * (180 * t + 20 * np.sin(2 * np.pi * t))) + 0.01 * rng.standard_normal(t.size)
    if quiet_stretch:
        x[s.block // 3:s.block // 2] *= 1e-4
    x = np.stack([x, 0.5 * x], 1).astype(np.float32)
    return [x[i * s.block:(i + 1) * s.block] for i in range(n_blocks)]


def copy_draws(dst, src, row=None):
    """session ``dst`` takes ``src``'s draws of each block instead of drawing its own: every static draw buffer dst
    declares (``draw_buffers``) is copied from src's buffer of that name.  With ``row``, src is batched and dst one
    session: dst takes src's row ``row`` into the leading part of its buffer, and SineGen's rand_ini (one draw for all
    rows) whole.  The copies hold the buffers, not the sessions, so no reference cycle is made."""
    from ddsp_svc_b200.realtime import RAND_INI
    pairs = {}
    for stage, entries in dst.draw_buffers.items():
        pairs[stage] = []
        for name, kind in entries:
            d, s = getattr(dst, name), getattr(src, name)
            if row is not None and kind != RAND_INI:
                s = s[row:row + 1]
                d = d[:, :s.shape[1]]
            assert d.shape == s.shape, (name, d.shape, s.shape)
            pairs[stage].append((d, s))
    dst._draw = lambda stage: [d.copy_(s) for d, s in pairs[stage]]
