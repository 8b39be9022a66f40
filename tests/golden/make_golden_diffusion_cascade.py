"""Generate tests/golden/diffusion_cascade_state_dicts.json: the parameter trees (keys and shapes, buffers included) of
the LIVE reference's Unit2Mel, Unit2Wav and Unit2WavFast (diffusion/vocoder.py:171-314), on the CPU, for small models
and the widths of configs/diffusion.yaml, diffusion-new.yaml and diffusion-fast.yaml, with and without use_pitch_aug,
n_spk > 1 and pcmer_norm.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_diffusion_cascade.py

diffusion/diffusion.py imports librosa.sequence, which it never uses; where librosa is not installed the generator puts
an empty stand-in module in its place before importing, as make_golden_diffusion.py does.
"""
import json
import os
import sys
import types
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "diffusion_cascade_state_dicts.json")

# name -> (class, constructor kwargs as the reference's load_model_vocoder passes them)
MODELS = OrderedDict([
    ("mel_small", ("Unit2Mel", dict(input_channel=256, n_spk=1, use_pitch_aug=False, out_dims=128, n_layers=2,
                                    n_chans=64, n_hidden=256))),
    ("mel_small_spk_aug", ("Unit2Mel", dict(input_channel=768, n_spk=3, use_pitch_aug=True, out_dims=128, n_layers=2,
                                            n_chans=64, n_hidden=256))),
    ("mel_diffusion_yaml", ("Unit2Mel", dict(input_channel=768, n_spk=1, use_pitch_aug=True, out_dims=128,
                                             n_layers=20, n_chans=512, n_hidden=256))),
    ("wav_small", ("Unit2Wav", dict(sampling_rate=44100, block_size=512, n_unit=256, n_spk=1, use_pitch_aug=False,
                                    out_dims=128, n_layers=2, n_chans=64, pcmer_norm=False))),
    ("wav_small_spk_aug_norm", ("Unit2Wav", dict(sampling_rate=44100, block_size=512, n_unit=256, n_spk=2,
                                                 use_pitch_aug=True, out_dims=128, n_layers=2, n_chans=64,
                                                 pcmer_norm=True))),
    ("wav_diffusion_new_yaml", ("Unit2Wav", dict(sampling_rate=44100, block_size=512, n_unit=768, n_spk=1,
                                                 use_pitch_aug=True, out_dims=128, n_layers=20, n_chans=512,
                                                 pcmer_norm=False))),
    ("fast_small", ("Unit2WavFast", dict(sampling_rate=44100, block_size=512, win_length=2048, n_unit=256, n_spk=1,
                                         use_pitch_aug=False, out_dims=128, n_layers=2, n_chans=128))),
    ("fast_small_spk_aug", ("Unit2WavFast", dict(sampling_rate=44100, block_size=512, win_length=2048, n_unit=256,
                                                 n_spk=2, use_pitch_aug=True, out_dims=128, n_layers=2, n_chans=128))),
    ("fast_diffusion_fast_yaml", ("Unit2WavFast", dict(sampling_rate=44100, block_size=512, win_length=2048,
                                                       n_unit=768, n_spk=1, use_pitch_aug=True, out_dims=128,
                                                       n_layers=6, n_chans=512))),
])


def _reference():
    from oracle import mel as omel
    omel.load_reference_stft()                       # the checkout on sys.path; nvSTFT's librosa stubbed where missing
    if not hasattr(sys.modules["librosa"], "sequence"):          # diffusion.py imports it and never uses it
        seq = types.ModuleType("librosa.sequence")
        sys.modules["librosa"].sequence = seq
        sys.modules["librosa.sequence"] = seq
    import diffusion.vocoder as dv
    return dv


def main():
    dv = _reference()
    out = OrderedDict()
    for name, (cls, kw) in MODELS.items():
        net = getattr(dv, cls)(**kw)
        out[name] = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    with open(PATH, "w") as f:
        json.dump(out, f)
    print("wrote", PATH, {k: len(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
