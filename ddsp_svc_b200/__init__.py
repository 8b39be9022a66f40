"""ddsp_svc_b200 -- H100 (sm_90a) kernels for the DDSP harmonic-plus-noise synthesis path of
yxlllc/DDSP-SVC, behind the reference's Sins / CombSub / CombSubFast / CombSubSuperFast / SineGen forward()
API.  See DESIGN.md for the path, its boundary and the kernels; include/b200ddsp.h for the C ABI.
"""
from . import _lib, frontend, loss, mel, ops, sharding, synthetic  # noqa: F401
from .frontend import Volume_Extractor  # noqa: F401
from .loss import RSSLoss  # noqa: F401
from .dropin import build_model, load_model, patch_reference, unpatch_reference  # noqa: F401
from .pipeline import HostPipeline  # noqa: F401
from .sinegen import SineGen, SourceModuleHnNSF  # noqa: F401
from .vocoder import CombSub, CombSubFast, CombSubSuperFast, FixedControls, Sins  # noqa: F401

__all__ = ["Sins", "CombSub", "CombSubSuperFast", "CombSubFast", "SineGen", "SourceModuleHnNSF", "FixedControls", "HostPipeline", "Volume_Extractor", "RSSLoss", "frontend", "loss", "mel", "ops", "synthetic", "sharding",
           "patch_reference", "unpatch_reference", "load_model", "build_model"]
