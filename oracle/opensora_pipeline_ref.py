"""TEST INFRASTRUCTURE ONLY -- loads the reference's OpenSora pipeline module (videosys/pipelines/open_sora/
pipeline_open_sora.py) and its data_process.py unmodified, so that their conditioning helpers (extract_json_from_prompts,
split_prompt / merge_prompt / extract_prompts_loop, parse_mask_strategy, find_nearest_point, apply_mask_strategy,
append_generated, dframe_to_frame, resize_crop_to_fill, read_image_from_path) run as written.

The module-level imports that are not installed, or not importable here, are stand-ins that those helpers never call:
ftfy and bs4 (prompt cleaning), diffusers' DiffusionPipeline and the videosys pipeline base class, videosys.utils.utils
(save_video, set_seed) and torchvision.io.write_video (gone from torchvision 0.26)."""
import importlib
import sys
import types

_LOADED = {}


def _stub(name, **kw):
    if name in sys.modules:
        return sys.modules[name]
    m = types.ModuleType(name)
    m.__dict__.update(kw)
    sys.modules[name] = m
    return m


def load():
    """(pipeline_open_sora, data_process) of the reference (cached)."""
    if _LOADED:
        return _LOADED["pipeline"], _LOADED["data"]
    from oracle import opensora_vae_ref, ref_loader

    ref_loader.load()
    opensora_vae_ref.load_opensora_vae()
    # ref_loader.load() installs a bare diffusers.models when it runs after the VAE module was cached: the pipeline
    # module imports AutoencoderKL from it (never called by the helpers)
    models = sys.modules["diffusers.models"]
    if not hasattr(models, "AutoencoderKL"):
        models.AutoencoderKL = opensora_vae_ref._AutoencoderKLStandIn
    for name in ("ftfy", "bs4"):
        try:
            importlib.import_module(name)
        except ImportError:
            _stub(name, BeautifulSoup=object)
    _stub("diffusers.pipelines")
    _stub("diffusers.pipelines.pipeline_utils", DiffusionPipeline=type("DiffusionPipeline", (), {}))
    _stub("videosys.core.pipeline.pipeline", VideoSysPipeline=type("VideoSysPipeline", (), {}), VideoSysPipelineOutput=object)
    _stub("videosys.utils.utils", save_video=None, set_seed=None)
    import torchvision.io

    if not hasattr(torchvision.io, "write_video"):
        torchvision.io.write_video = None
    _LOADED["pipeline"] = importlib.import_module("videosys.pipelines.open_sora.pipeline_open_sora")
    _LOADED["data"] = importlib.import_module("videosys.pipelines.open_sora.data_process")
    return _LOADED["pipeline"], _LOADED["data"]
