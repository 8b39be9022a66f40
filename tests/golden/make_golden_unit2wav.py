"""Generate tests/golden/unit2wav_*.npz: the LIVE reference's reflow cascade Unit2Wav.forward (reflow/vocoder.py:149-197:
CombSubSuperFast -> Vocoder.extract -> RectifiedFlow -> Vocoder.infer, NSF-HiFiGAN) on the CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT; librosa / soundfile stubbed as in make_golden_mel.py):

    python tests/golden/make_golden_unit2wav.py [case names; default: all]

Weights are not stored: ``state_dict`` / ``generator_state_dict`` rebuild them from a seed without the reference (the
package's Unit2Wav and Generator have the reference's trees): the DDSP model at its default init under
``torch.manual_seed``, the velocity network and the vocoder through tests/reflow_oracle.seeded_weights (every parameter
non-zero).  The vocoder is conversion_fixtures.HIFIGAN (44.1 kHz, hop 512, 128 mels).  unit2wav_state_dicts.json lists the
reference Unit2Wav's keys and shapes for each model.

Each file holds the inputs (units, f0, volume, spk_id, aug_shift), the case's settings, the reference's fp32 output
``out32`` and ``out64``, the same forward with the module, the inputs and the draws in float64 (the reference keeps
SineGen's phase increments in fp32 there, ``rad[..., -1:].float()``).  The draws are the ones the reference made under
``torch.manual_seed(seed)``, in its order: CombSubSuperFast's randn_like of the combtooth [B, n_frames 512], the
sampler's randn [B, 1, 128, T] (not when t_start >= 1), SineGen's rand_ini [1, 1, 9] with its first entry zeroed and its
randn_like of the sines [B, T 512, 9] (not when return_wav is False).  ``reflow_noise`` and ``rand_ini`` are stored;
the two long ones keep a check (``<name>_head``, the first 512 values, and ``<name>_sum``, the float64 sum) and
``draws`` regenerates them from torch's CPU generator and verifies them against it.
"""
import json
import os
import sys
import tempfile
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import reflow_oracle  # noqa: E402
from conversion_fixtures import HIFIGAN  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
N_UNIT, N_SPK, UPP = 256, 2, 512
MODELS = OrderedDict([("w128", dict(n_chans=128, n_layers=2, seed=61)), ("w512", dict(n_chans=512, n_layers=6, seed=62))])
VOCODER_SEED = 63

CASES = OrderedDict([
    ("unit2wav_w128_f24_euler3_t07", dict(model="w128", F=24, method="euler", steps=3, t_start=0.7, key=0.0,
                                          silence_front=0.0, return_wav=True)),
    ("unit2wav_w128_f30_rk4_2_key1p5_sf2", dict(model="w128", F=30, method="rk4", steps=2, t_start=0.7, key=1.5,
                                                silence_front=0.03, return_wav=True)),
    ("unit2wav_w128_f20_t1", dict(model="w128", F=20, method="euler", steps=3, t_start=1.0, key=0.0,
                                  silence_front=0.0, return_wav=True)),
    ("unit2wav_w128_f20_mel", dict(model="w128", F=20, method="euler", steps=3, t_start=0.7, key=-2.0,
                                   silence_front=0.0, return_wav=False)),
    ("unit2wav_w512_f16_euler3_t07", dict(model="w512", F=16, method="euler", steps=3, t_start=0.7, key=0.0,
                                          silence_front=0.0, return_wav=True)),
])


def path(name):
    return os.path.join(HERE, name + ".npz")


def _seed(name):
    return 6000 + list(CASES).index(name)


def state_dict(model):
    """the Unit2Wav state dict of a model: the DDSP model at its default init, the velocity network seeded"""
    import ddsp_svc_b200 as pkg
    m = MODELS[model]
    torch.manual_seed(m["seed"])
    net = pkg.Unit2Wav(HIFIGAN["sampling_rate"], HIFIGAN["hop_size"], 2048, N_UNIT, N_SPK, True, HIFIGAN["num_mels"],
                       m["n_layers"], m["n_chans"])
    reflow_oracle.seeded_weights(net.reflow_model.velocity_fn, m["seed"])
    return net.state_dict()


def generator_state_dict():
    """the vocoder's generator with weight norm attached, every parameter seeded"""
    import warnings
    from ddsp_svc_b200.dropin import DotDict
    from ddsp_svc_b200.hifigan import Generator
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen = Generator(DotDict(HIFIGAN))
    return reflow_oracle.seeded_weights(gen, VOCODER_SEED, gain=0.5).state_dict()


def write_vocoder(d):
    """config.json and model.ckpt of the vocoder in directory d -> the checkpoint's path"""
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(HIFIGAN, f)
    ckpt = os.path.join(d, "model.ckpt")
    torch.save({"generator": generator_state_dict()}, ckpt)
    return ckpt


def build_inputs(name):
    """units [1, F, 256], f0 [1, F, 1] (a glide with an unvoiced stretch), volume [1, F, 1], spk_id [1, 1],
    aug_shift [1, 1]"""
    c = CASES[name]
    g = torch.Generator().manual_seed(_seed(name))
    F_ = c["F"]
    t = torch.arange(F_, dtype=torch.float32) / F_
    f0 = 140 * 2 ** (t + 0.1 * torch.sin(6.0 * t))
    f0[F_ // 3:F_ // 3 + 3] = 0
    volume = 0.05 + 0.2 * torch.rand(F_, generator=g)
    return dict(units=torch.randn(1, F_, N_UNIT, generator=g), f0=f0[None, :, None], volume=volume[None, :, None],
                spk_id=torch.tensor([[1 + _seed(name) % N_SPK]]), aug_shift=torch.tensor([[c["key"]]]))


def draw_shapes(name):
    """(name, torch function, shape) of the reference's draws in its order"""
    c = CASES[name]
    T = c["F"] - int(c["silence_front"] * HIFIGAN["sampling_rate"] / HIFIGAN["hop_size"])
    out = [("ddsp_noise", "randn", (1, c["F"] * HIFIGAN["hop_size"]))]
    if c["t_start"] < 1.0:
        out.append(("reflow_noise", "randn", (1, 1, HIFIGAN["num_mels"], T)))
    if c["return_wav"]:
        out += [("rand_ini", "rand", (1, 1, 9)), ("sine_noise", "randn", (1, T * UPP, 9))]
    return out


def draws(d, name):
    """{draw name: tensor} of a golden file ``d``, regenerated from its seed in the reference's order and checked
    against what the reference drew"""
    g = torch.Generator().manual_seed(int(d["seed"]))
    out = {}
    for k, fn, shape in draw_shapes(name):
        v = getattr(torch, fn)(shape, generator=g)
        if k == "rand_ini":
            v[..., 0] = 0
        out[k] = v
        if k + "_sum" in d:
            ok = (np.array_equal(v.reshape(-1)[:512].numpy(), d[k + "_head"])
                  and v.double().sum().item() == float(d[k + "_sum"]))
        else:
            ok = np.array_equal(v.numpy(), d[k])
        if not ok:
            raise AssertionError("the regenerated %s differs from the one the reference drew" % k)
    return out


def _reference():
    from oracle import mel as omel
    from oracle import ref_loader
    ref_loader.load()
    omel.load_reference_stft()
    import reflow.vocoder as rv
    return rv


class _Draws:
    """records torch.randn / randn_like / rand while active (record=True), or returns the given tensors in order"""

    def __init__(self, replay=None):
        self.seen, self.replay = [], replay

    def __enter__(self):
        self.saved = {n: getattr(torch, n) for n in ("randn", "randn_like", "rand")}
        for n, f in self.saved.items():
            setattr(torch, n, self._wrap(f))
        return self

    def _wrap(self, f):
        def call(*a, **k):
            if self.replay is not None:
                v = self.replay[len(self.seen)]
                ref = f(*a, **k)
                assert tuple(v.shape) == tuple(ref.shape), (v.shape, ref.shape)
                v = v.to(ref.dtype).clone()
            else:
                v = f(*a, **k)
            self.seen.append(v)
            return v
        return call

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(torch, n, f)
        return False


def generate(name, voc_ckpt):
    c = CASES[name]
    rv = _reference()
    m = MODELS[c["model"]]
    net = rv.Unit2Wav(HIFIGAN["sampling_rate"], HIFIGAN["hop_size"], 2048, N_UNIT, N_SPK, True, HIFIGAN["num_mels"],
                      m["n_layers"], m["n_chans"])
    net.load_state_dict(state_dict(c["model"]), strict=True)
    net.eval()
    inp = build_inputs(name)
    kw = dict(infer=True, return_wav=c["return_wav"], infer_step=c["steps"], method=c["method"], t_start=c["t_start"],
              silence_front=c["silence_front"], use_tqdm=False)
    out = {k: v.numpy() for k, v in inp.items()}
    out.update(seed=np.array(_seed(name)), **{k: np.array(v) for k, v in c.items() if k != "model"})
    vocoder = rv.Vocoder("nsf-hifigan", voc_ckpt, device="cpu")
    # the generator is built now, not on first use: its init would draw from the seeded generator mid-forward
    from nsf_hifigan.models import load_model
    vocoder.vocoder.model, vocoder.vocoder.h = load_model(voc_ckpt, device="cpu")
    with torch.no_grad():
        torch.manual_seed(_seed(name))
        with _Draws() as rec:
            y32 = net(inp["units"], inp["f0"], inp["volume"], spk_id=inp["spk_id"], aug_shift=inp["aug_shift"],
                      vocoder=vocoder, **kw)
        shapes = draw_shapes(name)
        assert [tuple(v.shape) for v in rec.seen] == [s for _, _, s in shapes], [v.shape for v in rec.seen]
        recorded = {k: v for (k, _, _), v in zip(shapes, rec.seen)}
        for k, v in recorded.items():
            if k in ("ddsp_noise", "sine_noise"):
                out[k + "_head"] = v.reshape(-1)[:512].numpy()
                out[k + "_sum"] = np.array(v.double().sum().item())
            else:
                out[k] = v.numpy()
        out["out32"] = y32.numpy()
        # float64: the module, the inputs and the same draws in double (the mel basis is cached in double first)
        prev = torch.get_default_dtype()
        torch.set_default_dtype(torch.float64)
        try:
            net64 = net.double()
            vocoder.vocoder.model.double()
            stft = vocoder.vocoder.stft
            stft.mel_basis = {k: v.double() for k, v in stft.mel_basis.items()}
            stft.hann_window = {k: v.double() for k, v in stft.hann_window.items()}
            with _Draws(replay=list(rec.seen)):
                y64 = net64(inp["units"].double(), inp["f0"].double(), inp["volume"].double(), spk_id=inp["spk_id"],
                            aug_shift=inp["aug_shift"].double(), vocoder=vocoder, **kw)
        finally:
            torch.set_default_dtype(prev)
        out["out64"] = y64.numpy()
    assert draws(out, name)
    np.savez_compressed(path(name), **out)
    return out


def write_state_dict_keys():
    """unit2wav_state_dicts.json: [key, shape] of the reference's Unit2Wav for each model"""
    rv = _reference()
    sd = {}
    for model, m in MODELS.items():
        net = rv.Unit2Wav(HIFIGAN["sampling_rate"], HIFIGAN["hop_size"], 2048, N_UNIT, N_SPK, True,
                          HIFIGAN["num_mels"], m["n_layers"], m["n_chans"])
        sd[model] = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    with open(os.path.join(HERE, "unit2wav_state_dicts.json"), "w") as f:
        json.dump(sd, f)


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    write_state_dict_keys()
    with tempfile.TemporaryDirectory() as d:
        ckpt = write_vocoder(d)
        for n in names:
            o = generate(n, ckpt)
            a, b = o["out32"].astype(np.float64), o["out64"]
            print("wrote", path(n), o["out32"].shape, "reference fp32 rel rms %.2e" %
                  (np.sqrt(np.mean((a - b) ** 2)) / np.sqrt(np.mean(b ** 2))))
