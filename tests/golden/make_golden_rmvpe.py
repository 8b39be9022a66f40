"""Generate tests/golden/rmvpe_*.npz and rmvpe_state_dicts.json: the LIVE reference's RMVPE (encoder/rmvpe/) on the CPU.

Needs a reference checkout (DDSP_REFERENCE_ROOT):

    python tests/golden/make_golden_rmvpe.py [case names; default: all]

Weights are not stored: ``model(name)`` rebuilds them from a seed (tests/rmvpe_oracle.seeded_model: default init under
``torch.manual_seed``, BatchNorm calibrated by one train-mode pass in float64).  Each file keeps ``weights_sum``, the
float64 sum of every floating tensor of that state dict, which ``model`` checks before a test uses the weights.
rmvpe_state_dicts.json holds the reference's key / shape tree of each model.

Network cases hold the log-mel ``mel`` [B, 128, n] and, from the reference's ``RMVPE.mel2hidden`` (padding to a multiple of
32 frames, ``E2E0.forward``, crop), ``hidden64`` (the module in float64) and ``hidden32`` (fp32), with
``to_local_average_f0`` of each, ``f0_64`` and ``f0_32``.  Audio cases hold seeded audio at ``sr`` whose length is not a
multiple of 441: ``f0_32`` is ``RMVPE.infer_from_audio`` itself (fp32 on the CPU); ``hidden64`` / ``f0_64`` are its
pieces in float64 (torchaudio Resample, spec.py's MelSpectrogram, mel2hidden, to_local_average_f0).  Every case asserts
that the salience is not saturated: at least half its entries in (0.01, 0.99).

Where librosa is absent, the shared stub (oracle/mel.py) answers ``librosa.filters.mel`` with the Slaney basis whatever
``htk`` says.  spec.py asks for ``htk=True``, so ``reference()`` hands spec.py an HTK basis of its own, built from
torchaudio's ``melscale_fbanks(mel_scale='htk', norm='slaney')`` in float64 (not from the package under test), and checks
that the reference's MelSpectrogram really holds it.
"""
import json
import os
import sys
import tempfile
import types
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from tests import rmvpe_oracle as ro  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
MODELS = OrderedDict([("full", dict(cfg=dict(), seed=0)),
                      ("reduced", dict(cfg=dict(n_blocks=1, en_de_layers=2, inter_layers=1), seed=7))])
CASES = OrderedDict()
for _B, _n in ((1, 1), (2, 31), (1, 32), (2, 33), (1, 100)):
    CASES["rmvpe_full_b%d_n%d" % (_B, _n)] = dict(model="full", B=_B, n=_n)
CASES["rmvpe_reduced_b1_n160"] = dict(model="reduced", B=1, n=160)
CASES["rmvpe_audio_44100"] = dict(model="full", sr=44100, N=44100 // 2 + 123)
CASES["rmvpe_audio_16000"] = dict(model="full", sr=16000, N=8000 + 77)


def path(name):
    return os.path.join(HERE, name + ".npz")


def _seed(name):
    return 5000 + list(CASES).index(name)


def htk_basis(sr, n_fft, n_mels=128, fmin=0.0, fmax=None):
    """librosa.filters.mel(..., htk=True) (norm 'slaney', float32) through torchaudio's melscale_fbanks in float64"""
    import torchaudio
    fmax = sr / 2 if fmax is None else fmax
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        fb = torchaudio.functional.melscale_fbanks(n_fft // 2 + 1, float(fmin), float(fmax), n_mels, sr, norm="slaney",
                                                   mel_scale="htk")
    finally:
        torch.set_default_dtype(prev)
    return fb.T.numpy().astype(np.float32)


def reference():
    """the reference's encoder.rmvpe package, importable without librosa (see the module docstring)"""
    ref_loader.load()
    from oracle import mel as om
    om.load_reference_stft()                       # the shared librosa stub, where librosa is absent
    lib = sys.modules["librosa"]
    stub = getattr(lib, "__b2d_stub__", False)
    if stub and "librosa.sequence" not in sys.modules:
        seq = types.ModuleType("librosa.sequence")   # utils.py imports librosa; only Viterbi decoding uses it
        sys.modules["librosa.sequence"] = seq
        lib.sequence = seq
    import encoder.rmvpe as rm
    import encoder.rmvpe.spec as spec
    if stub:
        def mel(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, htk=False, **unused):
            if not htk:
                raise NotImplementedError("only spec.py's htk=True basis is provided here")
            return htk_basis(sr, n_fft, n_mels, fmin, fmax)
        spec.mel = mel
    probe = rm.MelSpectrogram(128, 16000, 1024, 160, None, 30, 8000)
    assert np.abs(probe.mel_basis.numpy() - htk_basis(16000, 1024, 128, 30, 8000)).max() < 1e-6, \
        "the reference's MelSpectrogram does not hold the HTK basis spec.py asks for"
    return rm


def weights_sum(sd):
    return float(sum(v.double().sum() for v in sd.values() if v.is_floating_point()))


def model(name, expected_sum=None):
    """the seeded E2E0 (ddsp_svc_b200.E2E0, fp32, eval) of MODELS[name]; checks ``expected_sum`` when given"""
    spec = MODELS[name]
    with torch.no_grad():
        m = ro.seeded_model(seed=spec["seed"], **spec["cfg"])
    if expected_sum is not None:
        got = weights_sum(m.state_dict())
        assert abs(got - expected_sum) <= 1e-9 * max(1.0, abs(expected_sum)), (got, expected_sum)
    return m


def load(name):
    """the golden of case ``name`` as a dict of numpy arrays / scalars, and its model with the weights checked"""
    with np.load(path(name)) as z:
        d = {k: z[k] for k in z.files}
    return d, model(str(d["model"]), float(d["weights_sum"]))


def _unsaturated(h, name):
    frac = float(((h > 0.01) & (h < 0.99)).mean())
    assert frac >= 0.5, "%s: salience saturated (%.3f of entries in (0.01, 0.99))" % (name, frac)


def make(name, rm, models):
    c = CASES[name]
    ours, ref32, sd = models[c["model"]]
    from encoder.rmvpe.utils import to_local_average_f0
    ref64 = type(ref32)(*ref32._b2d_args).double().eval()
    ref64.load_state_dict(ref32.state_dict())
    g = torch.Generator().manual_seed(_seed(name))
    out = dict(model=np.array(c["model"]), weights_sum=np.float64(weights_sum(sd)), seed=np.int64(_seed(name)))
    pad = lambda x: torch.nn.functional.pad(x, (0, 32 * ((x.shape[-1] - 1) // 32 + 1) - x.shape[-1]))
    with torch.no_grad():
        if "sr" in c:
            sr, N = c["sr"], c["N"]
            audio = (0.3 * torch.sin(2 * np.pi * 220.0 * torch.arange(N, dtype=torch.float64) / sr)
                     + 0.02 * torch.randn(N, generator=g, dtype=torch.float64)).float()
            with tempfile.TemporaryDirectory() as tmp:
                ckpt = os.path.join(tmp, "model.pt")
                torch.save({"model": sd}, ckpt)
                ex = rm.RMVPE(ckpt, hop_length=160)
            f0_32 = ex.infer_from_audio(audio.numpy(), sample_rate=sr, device="cpu", thred=0.03, use_viterbi=False)
            import torchaudio
            a64 = audio.double()[None]
            if sr != 16000:
                a64 = torchaudio.transforms.Resample(sr, 16000, lowpass_filter_width=128).double()(a64)
            mel64 = rm.MelSpectrogram(128, 16000, 1024, 160, None, 30, 8000).double()(a64, center=True)
            n = mel64.shape[-1]
            h64 = ref64(pad(mel64))[:, :n]
            out.update(sr=np.int64(sr), audio=audio.numpy(), f0_32=np.asarray(f0_32, np.float32)[None],
                       hidden64=h64.numpy(), f0_64=np.asarray(to_local_average_f0(h64, thred=0.03))[None])
        else:
            B, n = c["B"], c["n"]
            mel = (torch.randn(B, 128, n, generator=g, dtype=torch.float64) - 4.0).float()
            h64 = ref64(pad(mel.double()))[:, :n]
            h32 = ref32(pad(mel))[:, :n]
            f0_64 = np.asarray(to_local_average_f0(h64, thred=0.03)).reshape(B, n)
            f0_32 = np.asarray(to_local_average_f0(h32, thred=0.03)).reshape(B, n)
            out.update(mel=mel.numpy(), hidden64=h64.numpy(), hidden32=h32.numpy(), f0_64=f0_64, f0_32=f0_32)
    _unsaturated(out["hidden64"], name)
    np.savez(path(name), **out)
    assert os.path.getsize(path(name)) < 1 << 20, name
    print("wrote", path(name), os.path.getsize(path(name)), "bytes")


def main(names):
    torch.set_num_threads(1)                       # a fixed summation order: byte-identical regeneration
    rm = reference()
    models, trees = {}, {}
    args = {"full": (4, 1, (2, 2)), "reduced": (1, 1, (2, 2), 2, 1)}
    for mname in MODELS:
        ours = model(mname)
        sd = ours.state_dict()
        ref32 = rm.E2E0(*args[mname]).eval()
        ref32._b2d_args = args[mname]
        ref32.load_state_dict(sd, strict=True)
        models[mname] = (ours, ref32, sd)
        trees[mname] = OrderedDict((k, list(v.shape)) for k, v in ref32.state_dict().items())
    with open(os.path.join(HERE, "rmvpe_state_dicts.json"), "w") as f:
        json.dump(trees, f, separators=(",", ":"))
    for name in names or CASES:
        make(name, rm, models)


if __name__ == "__main__":
    main(sys.argv[1:])
