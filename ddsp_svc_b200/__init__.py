"""ddsp_svc_b200 -- H100 (sm_90a) kernels for the DDSP harmonic-plus-noise synthesis path of
yxlllc/DDSP-SVC, behind the reference's Sins / CombSub / CombSubFast / CombSubSuperFast / SineGen / NSF-HiFiGAN
Generator forward() API, the diffusion / reflow models' NSF-HiFiGAN Vocoder, the RMVPE pitch extractor and the HuBERT /
ContentVec units encoders.  See DESIGN.md for the path, its boundary and the kernels; include/b200ddsp.h for the C ABI.
"""
from . import _lib, frontend, loss, mel, ops, sharding, synthetic  # noqa: F401
from .frontend import Volume_Extractor  # noqa: F401
from .enhancer import Enhancer  # noqa: F401
from .hifigan import Generator  # noqa: F401
from .hubert import HubertSoft, Units_Encoder, load_fairseq_hubert  # noqa: F401
from .nsf_vocoder import Vocoder  # noqa: F401
from .loss import RSSLoss  # noqa: F401
from .diffusion import GaussianDiffusion, WaveNet  # noqa: F401
from .diffusion_vocoder import DiffGtMel, Unit2Mel, Unit2WavFast  # noqa: F401
from .dropin import build_model, load_model, patch_reference, unpatch_reference  # noqa: F401
from .offline import OfflineDiffVC, OfflineReflowVC, OfflineVC  # noqa: F401
from .pipeline import HostPipeline  # noqa: F401
from .realtime import BatchedRealtimeVC, RealtimeDiffVC, RealtimeReflowVC, RealtimeVC  # noqa: F401
from .reflow import NaiveV2Diff, RectifiedFlow  # noqa: F401
from .reflow_vocoder import Unit2Wav, load_model_vocoder  # noqa: F401
from .rmvpe import E2E0, RMVPE  # noqa: F401
from .sinegen import SineGen, SourceModuleHnNSF  # noqa: F401
from .vocoder import CombSub, CombSubFast, CombSubSuperFast, FixedControls, Sins  # noqa: F401

__all__ = ["Sins", "CombSub", "CombSubSuperFast", "CombSubFast", "SineGen", "SourceModuleHnNSF", "FixedControls", "HostPipeline", "RealtimeVC", "BatchedRealtimeVC", "RealtimeReflowVC", "RealtimeDiffVC", "OfflineVC", "OfflineReflowVC", "OfflineDiffVC", "NaiveV2Diff", "RectifiedFlow", "Unit2Wav", "Unit2Mel", "Unit2WavFast", "DiffGtMel", "WaveNet", "GaussianDiffusion", "Generator", "E2E0", "RMVPE", "HubertSoft", "Units_Encoder", "load_fairseq_hubert", "Vocoder", "Enhancer", "Volume_Extractor", "RSSLoss", "frontend", "loss", "mel", "ops", "synthetic", "sharding",
           "patch_reference", "unpatch_reference", "load_model", "build_model", "load_model_vocoder"]
