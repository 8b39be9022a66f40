"""Import the upstream reference (yxlllc/DDSP-SVC) for oracle validation.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  The reference is a Python /
PyTorch program; its hot path (ddsp/vocoder.py, ddsp/core.py,
nsf_hifigan/models.py) imports several third-party packages that are not
installed here and are not used by the path.  They are replaced by empty stub
modules before import.  The reference is not part of this repository: point
DDSP_REFERENCE_ROOT at a checkout of it to use it (the golden generators under
tests/golden/ need it); callers must check ``available()`` first.
"""
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("DDSP_REFERENCE_ROOT", "")

_STUBS = ("pyworld", "parselmouth", "torchcrepe", "resampy", "fairseq", "gin",
          "local_attention")


def available() -> bool:
    return bool(REFERENCE_ROOT) and os.path.isfile(os.path.join(REFERENCE_ROOT, "ddsp", "vocoder.py"))


def _install_stubs():
    for name in _STUBS:
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["fairseq"].checkpoint_utils = types.SimpleNamespace()
    sys.modules["local_attention"].LocalAttention = object
    if "matplotlib" not in sys.modules:
        try:
            import matplotlib  # noqa: F401
        except Exception:
            mpl = types.ModuleType("matplotlib")
            mpl.use = lambda *a, **k: None
            sys.modules["matplotlib"] = mpl
            for sub in ("pylab", "pyplot"):
                sys.modules["matplotlib." + sub] = types.ModuleType("matplotlib." + sub)


_cache = {}


def load():
    """Return (ddsp.vocoder module, ddsp.core module, nsf_hifigan.models.SineGen)."""
    if "mods" in _cache:
        return _cache["mods"]
    if not available():
        raise RuntimeError("reference not found: set DDSP_REFERENCE_ROOT to a DDSP-SVC checkout")
    sys.dont_write_bytecode = True  # the reference checkout may be read-only
    _install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import ddsp.vocoder as V
    import ddsp.core as C
    from nsf_hifigan.models import SineGen
    _cache["mods"] = (V, C, SineGen)
    return _cache["mods"]


def fixed_ctrl_module(ctrls, hidden):
    """A torch module standing in for Unit2Control: returns fixed raw controls.

    This is the DSP/NN seam of the reference (ddsp/vocoder.py:578, :664, :832).
    """
    import torch

    class FixedCtrl(torch.nn.Module):
        def forward(self, *a, **k):
            return ctrls, hidden

    return FixedCtrl()
