"""Drop-in wiring for an existing DDSP-SVC checkout.

``patch_reference()`` rebinds the reference's synthesizer classes to this package's ones so that its
unmodified entry points (main.py, flask_api.py, gui.py, enhancer.py, ...) run on the CUDA
kernels:

    import ddsp_svc_b200
    ddsp_svc_b200.patch_reference()      # before `from ddsp.vocoder import load_model`
    # ... the rest of main.py unchanged

``load_model`` mirrors the reference's ``ddsp/vocoder.py:475-529`` (config.yaml next to the
checkpoint -> class dispatch -> strict load_state_dict) for use without patching.
"""
import os
import sys

import torch
import yaml

from . import sinegen, vocoder


class DotDict(dict):
    """Attribute access to nested config dicts (same behaviour as the reference's DotDict,
    ddsp/vocoder.py:467-473 / logger/utils.py:49-56)."""

    def __getattr__(self, key):
        val = self.get(key)
        return DotDict(val) if type(val) is dict else val

    __setattr__ = dict.__setitem__
    __delattr__ = dict.__delitem__


_MODEL_TYPES = {
    "Sins": lambda a: vocoder.Sins(
        sampling_rate=a.data.sampling_rate, block_size=a.data.block_size, n_harmonics=a.model.n_harmonics,
        n_mag_allpass=a.model.n_mag_allpass, n_mag_noise=a.model.n_mag_noise,
        n_unit=a.data.encoder_out_channels, n_spk=a.model.n_spk),
    "CombSub": lambda a: vocoder.CombSub(
        sampling_rate=a.data.sampling_rate, block_size=a.data.block_size, n_mag_allpass=a.model.n_mag_allpass,
        n_mag_harmonic=a.model.n_mag_harmonic, n_mag_noise=a.model.n_mag_noise,
        n_unit=a.data.encoder_out_channels, n_spk=a.model.n_spk),
    "CombSubFast": lambda a: vocoder.CombSubFast(
        sampling_rate=a.data.sampling_rate, block_size=a.data.block_size,
        n_unit=a.data.encoder_out_channels, n_spk=a.model.n_spk),
    "CombSubSuperFast": lambda a: vocoder.CombSubSuperFast(
        sampling_rate=a.data.sampling_rate, block_size=a.data.block_size, win_length=a.model.win_length,
        n_unit=a.data.encoder_out_channels, n_spk=a.model.n_spk),
}


def build_model(args):
    """Config (DotDict) -> synthesizer module; unknown types raise like the reference (:522)."""
    make = _MODEL_TYPES.get(args.model.type)
    if make is None:
        raise ValueError(f" [x] Unknown Model: {args.model.type}")
    return make(args)


def load_model(model_path, device="cuda"):
    config_file = os.path.join(os.path.split(model_path)[0], "config.yaml")
    with open(config_file, "r") as config:
        args = DotDict(yaml.safe_load(config))
    model = build_model(args)
    print(" [Loading] " + model_path)
    ckpt = torch.load(model_path, map_location=torch.device(device))
    model.to(device)
    model.load_state_dict(ckpt["model"])
    model.eval()
    return model, args


_REFLOW_MODULES = ("reflow.vocoder", "reflow.naive_v2_diff", "reflow.reflow")


def _patch_reflow(saved):
    """rebind NaiveV2Diff / RectifiedFlow in the reference's reflow modules (those that import); originals into saved"""
    import importlib
    from . import reflow as own
    for modname in _REFLOW_MODULES:
        try:
            mod = importlib.import_module(modname)
        except ImportError as e:
            saved.setdefault("_not_patched", {})[modname] = "%s: %s" % (type(e).__name__, e)
            continue
        for name in ("NaiveV2Diff", "RectifiedFlow"):
            if hasattr(mod, name):
                saved.setdefault(name, getattr(mod, name))
                setattr(mod, name, getattr(own, name))


_DIFFUSION_MODULES = ("diffusion.vocoder", "diffusion.diffusion", "diffusion.wavenet", "diffusion.naive_v2_diff")
_DIFFUSION_CLASSES = ("GaussianDiffusion", "WaveNet", "NaiveV2Diff")


def _patch_diffusion(saved):
    """rebind GaussianDiffusion / WaveNet / NaiveV2Diff in the reference's diffusion modules (those that import);
    originals into saved["diffusion"] by module, since NaiveV2Diff also has a reflow original"""
    import importlib
    from . import diffusion as own
    from . import reflow as own_reflow
    ours = dict(GaussianDiffusion=own.GaussianDiffusion, WaveNet=own.WaveNet, NaiveV2Diff=own_reflow.NaiveV2Diff)
    for modname in _DIFFUSION_MODULES:
        try:
            mod = importlib.import_module(modname)
        except ImportError as e:
            saved.setdefault("_not_patched", {})[modname] = "%s: %s" % (type(e).__name__, e)
            continue
        for name in _DIFFUSION_CLASSES:
            if hasattr(mod, name):
                saved.setdefault("diffusion", {}).setdefault(modname, {})[name] = getattr(mod, name)
                setattr(mod, name, ours[name])


_RMVPE_MODULES = ("encoder.rmvpe", "encoder.rmvpe.inference", "encoder.rmvpe.model")


def _patch_rmvpe(saved):
    """rebind RMVPE / E2E0 in the reference's encoder.rmvpe modules; originals into saved["rmvpe"] by module"""
    import importlib
    from . import rmvpe as own
    try:
        mods = [importlib.import_module(m) for m in _RMVPE_MODULES]
    except ImportError as e:                    # encoder.rmvpe imports librosa
        saved.setdefault("_not_patched", {})["encoder.rmvpe"] = "%s: %s" % (type(e).__name__, e)
        return
    import ddsp.vocoder as ref_vocoder
    cached = getattr(ref_vocoder, "F0_KERNEL", {}).get("rmvpe")
    if cached is not None and not isinstance(cached, own.RMVPE):
        saved.setdefault("_not_patched", {})["ddsp.vocoder.F0_KERNEL['rmvpe']"] = (
            "already holds a reference RMVPE instance; F0_Extractor keeps using it")
    for modname, mod in zip(_RMVPE_MODULES, mods):
        for name in ("RMVPE", "E2E0"):
            if hasattr(mod, name):
                saved.setdefault("rmvpe", {}).setdefault(modname, {})[name] = getattr(mod, name)
                setattr(mod, name, getattr(own, name))


def _patch_units(saved):
    """rebind Units_Encoder in ddsp.vocoder and HubertSoft in encoder.hubert.model and ddsp.vocoder; originals into
    saved["units"] by module"""
    import ddsp.vocoder as ref_vocoder
    from . import hubert as own
    targets = [(ref_vocoder, ("Units_Encoder", "HubertSoft"))]
    try:
        import encoder.hubert.model as ref_hubert
        targets.append((ref_hubert, ("HubertSoft",)))
    except ImportError as e:                    # encoder.hubert.model imports sklearn
        saved.setdefault("_not_patched", {})["encoder.hubert.model"] = "%s: %s" % (type(e).__name__, e)
    for mod, names in targets:
        for name in names:
            if hasattr(mod, name):
                saved.setdefault("units", {}).setdefault(mod.__name__, {})[name] = getattr(mod, name)
                setattr(mod, name, getattr(own, name))


_VOCODER_MODULES = ("diffusion.vocoder", "reflow.vocoder")


def _patch_vocoder(saved):
    """rebind Vocoder in the reference's diffusion.vocoder and reflow.vocoder (those that import); originals into
    saved["vocoder"] by module"""
    import importlib
    from .nsf_vocoder import Vocoder
    for modname in _VOCODER_MODULES:
        try:
            mod = importlib.import_module(modname)
        except ImportError as e:
            saved.setdefault("_not_patched", {})[modname] = "%s: %s" % (type(e).__name__, e)
            continue
        if hasattr(mod, "Vocoder"):
            saved.setdefault("vocoder", {}).setdefault(modname, {})["Vocoder"] = mod.Vocoder
            mod.Vocoder = Vocoder


def _patch_enhancer(saved):
    """rebind Enhancer in the reference's enhancer module; the original into saved["enhancer"]"""
    try:
        import enhancer as ref_enhancer
    except ImportError as e:
        saved.setdefault("_not_patched", {})["enhancer"] = "%s: %s" % (type(e).__name__, e)
        return
    from .enhancer import Enhancer
    saved.setdefault("enhancer", {})["enhancer"] = {"Enhancer": ref_enhancer.Enhancer}
    ref_enhancer.Enhancer = Enhancer


def patch_reference(reflow=False, diffusion=False, hifigan=False, rmvpe=False, units=False, vocoder=False,
                    enhancer=False):
    """Swap the synthesizer classes inside the (importable) reference package.  Returns the dict
    of original classes so a caller can restore them; its keys say what was patched.  If the enhancer stack
    (nsf_hifigan.models) cannot be imported, only the synthesizers are patched and the reason is returned under
    ``"_not_patched"`` -- any other failure propagates.

    ``reflow=True`` also rebinds the reflow model's velocity network and sampler (``NaiveV2Diff``, ``RectifiedFlow``)
    in reflow.vocoder, reflow.naive_v2_diff and reflow.reflow, so Unit2Wav samples on the kernels; a module that does not
    import is reported under ``"_not_patched"``.  Off by default.  To run train_reflow.py on the kernels, also set
    ``ddsp_svc_b200.NaiveV2Diff.reflow_backward = True``: then ``RectifiedFlow(infer=False)`` returns the reflow loss
    with its backward, and Unit2Wav's training step trains every parameter (INTEGRATION.md section 3b); without it
    infer=False and the sampler under grad raise NotImplementedError.

    ``diffusion=True`` rebinds the diffusion models' sampler and denoisers (``GaussianDiffusion``, ``WaveNet``,
    ``NaiveV2Diff``) in diffusion.vocoder, diffusion.diffusion, diffusion.wavenet and diffusion.naive_v2_diff, so
    Unit2Mel / Unit2Wav / Unit2WavFast (main_diff.py) sample on the kernels; a module that does not import (diffusion.diffusion
    imports librosa.sequence) is reported under ``"_not_patched"``.  Off by default.  To run train_diff.py on the kernels,
    also set ``ddsp_svc_b200.WaveNet.diffusion_backward = True`` (diffusion.yaml, diffusion-new.yaml) or
    ``ddsp_svc_b200.NaiveV2Diff.reflow_backward = True`` (diffusion-fast.yaml): then ``GaussianDiffusion(infer=False)``
    returns the diffusion loss with its backward (DESIGN.md section 4.15b); without them infer=False and calls under
    grad raise NotImplementedError.  The samplers under grad raise in any case.

    ``hifigan=True`` rebinds ``nsf_hifigan.models.Generator`` to ``ddsp_svc_b200.Generator``.  ``load_model`` looks the
    name up when it is called, so the enhancer (enhancer.py) and the diffusion and reflow vocoders (diffusion/vocoder.py,
    reflow/vocoder.py), which import ``load_model`` by name, all build the package's generator and vocode on the kernels.
    Off by default; needs nsf_hifigan.models to import (reported under ``"_not_patched"`` otherwise).

    ``rmvpe=True`` rebinds ``RMVPE`` and ``E2E0`` in encoder.rmvpe, encoder.rmvpe.inference and encoder.rmvpe.model to
    ``ddsp_svc_b200.RMVPE`` / ``ddsp_svc_b200.E2E0``.  F0_Extractor imports ``RMVPE`` from encoder.rmvpe when it first
    builds the 'rmvpe' extractor, so it then extracts f0 on the kernels.  Off by default.  If encoder.rmvpe does not
    import (it imports librosa), or ddsp.vocoder.F0_KERNEL['rmvpe'] already holds a reference instance (which
    F0_Extractor would keep using), that is reported under ``"_not_patched"``.

    ``units=True`` rebinds ``Units_Encoder`` in ddsp.vocoder and ``HubertSoft`` in ddsp.vocoder and encoder.hubert.model
    to ``ddsp_svc_b200.Units_Encoder`` / ``ddsp_svc_b200.HubertSoft``, so main.py, the GUIs, the APIs and preprocess.py
    encode units on the kernels ('hubertsoft', the 'hubertbase*' and the 'contentvec*' encoders; fairseq checkpoints
    load without fairseq).  Off by default.  If encoder.hubert.model does not import, that is reported under
    ``"_not_patched"``.

    ``vocoder=True`` rebinds ``Vocoder`` in diffusion.vocoder and reflow.vocoder to ``ddsp_svc_b200.Vocoder``, so
    preprocess.py extracts its mels, the pitch-augmented ones included, and train_diff.py / main_diff.py extract and
    vocode on the kernels.  preprocess.py and train_diff.py import ``Vocoder`` by name: patch before importing them.
    Off by default; a module that does not import is reported under ``"_not_patched"``.

    ``enhancer=True`` rebinds ``Enhancer`` in the reference's enhancer module to ``ddsp_svc_b200.enhancer.Enhancer``:
    resampling, f0 regridding, mel and vocoder on the kernels, and no host round trip for a numeric adaptive key.
    main.py and the GUIs import ``Enhancer`` by name: patch before importing them.  Off by default; if the module does
    not import, that is reported under ``"_not_patched"``."""
    import ddsp.vocoder as ref_vocoder          # the reference checkout must be on sys.path
    from . import vocoder as synths             # (the argument `vocoder` hides the module name here)
    names = ("Sins", "CombSub", "CombSubSuperFast", "CombSubFast")
    saved = {name: getattr(ref_vocoder, name) for name in names}
    for name in names:
        setattr(ref_vocoder, name, getattr(synths, name))
    from . import frontend                      # Volume_Extractor (numpy in -> numpy out like the reference, computed on the GPU)
    saved["Volume_Extractor"] = ref_vocoder.Volume_Extractor
    ref_vocoder.Volume_Extractor = frontend.Volume_Extractor
    try:                                        # mel front end of the enhancer / diffusion vocoders (needs librosa to import)
        import nsf_hifigan.nvSTFT as ref_stft
        from . import mel
        saved["STFT"] = ref_stft.STFT
        ref_stft.STFT = mel.STFT
    except ImportError as e:
        saved.setdefault("_not_patched", {})["nsf_hifigan.nvSTFT"] = "%s: %s" % (type(e).__name__, e)
    try:
        import nsf_hifigan.models as ref_nsf
    except ImportError as e:                    # enhancer stack not importable: synthesizers only (reported below)
        saved.setdefault("_not_patched", {})["nsf_hifigan.models"] = "%s: %s" % (type(e).__name__, e)
        ref_nsf = None
    if ref_nsf is not None:
        saved["SineGen"] = ref_nsf.SineGen
        saved["SourceModuleHnNSF"] = ref_nsf.SourceModuleHnNSF
        ref_nsf.SineGen = sinegen.SineGen
        ref_nsf.SourceModuleHnNSF = sinegen.SourceModuleHnNSF
        if hifigan:
            from .hifigan import Generator
            saved["Generator"] = ref_nsf.Generator
            ref_nsf.Generator = Generator
    if reflow:
        _patch_reflow(saved)
    if diffusion:
        _patch_diffusion(saved)
    if rmvpe:
        _patch_rmvpe(saved)
    if units:
        _patch_units(saved)
    if vocoder:
        _patch_vocoder(saved)
    if enhancer:
        _patch_enhancer(saved)
    return saved


def unpatch_reference(saved):
    import ddsp.vocoder as ref_vocoder
    for name in ("Sins", "CombSub", "CombSubSuperFast", "CombSubFast", "Volume_Extractor"):
        if name in saved:
            setattr(ref_vocoder, name, saved[name])
    if "STFT" in saved:
        import nsf_hifigan.nvSTFT as ref_stft
        ref_stft.STFT = saved["STFT"]
    if "SineGen" in saved:
        import nsf_hifigan.models as ref_nsf
        ref_nsf.SineGen = saved["SineGen"]
        if "SourceModuleHnNSF" in saved:
            ref_nsf.SourceModuleHnNSF = saved["SourceModuleHnNSF"]
        if "Generator" in saved:
            ref_nsf.Generator = saved["Generator"]
    if "NaiveV2Diff" in saved or "RectifiedFlow" in saved:
        for modname in _REFLOW_MODULES:
            mod = sys.modules.get(modname)
            for name in ("NaiveV2Diff", "RectifiedFlow"):
                if mod is not None and name in saved and hasattr(mod, name):
                    setattr(mod, name, saved[name])
    for modname, originals in (list(saved.get("diffusion", {}).items()) + list(saved.get("rmvpe", {}).items())
                               + list(saved.get("units", {}).items()) + list(saved.get("vocoder", {}).items())
                               + list(saved.get("enhancer", {}).items())):
        mod = sys.modules.get(modname)
        if mod is not None:
            for name, cls in originals.items():
                setattr(mod, name, cls)
