"""vsb200: the VideoSys DiT denoising hot path, H100-native (sm_90a CUDA behind a C-ABI).

Same top-level names as ``videosys/__init__.py:1-22`` for the paths in scope (OpenSora, CogVideoX, Latte, Vchitect, Open-Sora-Plan v1.1.0); see DESIGN.md.
"""
from .core.distributed.parallel_mgr import initialize  # noqa: F401
from .core.engine.engine import VideoSysEngine  # noqa: F401
from .core.pab.pab_mgr import PABConfig  # noqa: F401
from .pipelines.cogvideox.pipeline_cogvideox import CogVideoXConfig, CogVideoXPABConfig, CogVideoXPipeline  # noqa: F401
from .pipelines.latte.pipeline_latte import LatteConfig, LattePABConfig, LattePipeline  # noqa: F401
from .pipelines.open_sora.pipeline_open_sora import OpenSoraConfig, OpenSoraPABConfig, OpenSoraPipeline  # noqa: F401
from .pipelines.open_sora_plan.pipeline_open_sora_plan import (  # noqa: F401
    OpenSoraPlanConfig,
    OpenSoraPlanPipeline,
    OpenSoraPlanV110PABConfig,
    OpenSoraPlanV120PABConfig,
)
from .pipelines.vchitect.pipeline_vchitect import VchitectConfig, VchitectPABConfig, VchitectXLPipeline  # noqa: F401

__all__ = ["initialize", "VideoSysEngine", "PABConfig", "OpenSoraConfig", "OpenSoraPABConfig", "OpenSoraPipeline",
           "CogVideoXConfig", "CogVideoXPABConfig", "CogVideoXPipeline", "LatteConfig", "LattePABConfig", "LattePipeline", "OpenSoraPlanConfig",
           "OpenSoraPlanPipeline", "OpenSoraPlanV110PABConfig", "OpenSoraPlanV120PABConfig", "VchitectConfig", "VchitectPABConfig",
           "VchitectXLPipeline"]
