"""TEST INFRASTRUCTURE ONLY -- loads the reference's Open-Sora-Plan causal VAEs
(videosys/models/autoencoders/autoencoder_kl_open_sora_plan_v110.py and _v120.py) unmodified, on the reference checkout
that oracle/ref_loader.py finds.

Their diffusers imports are mixins (``ModelMixin``, ``ConfigMixin``, ``register_to_config``) and ``logging``; they are
replaced by the stand-ins of oracle/cogvideox_vae_ref.py plus a no-op ``logging``.  torchvision, huggingface_hub and einops
are the installed packages (the hub is never reached: the models are built from keywords).
"""
import importlib
import types

import torch.nn as nn

from oracle import cogvideox_vae_ref as C
from oracle import ref_loader

_LOADED = {}


def load_osp_vae(version):
    """The reference module ``videosys.models.autoencoders.autoencoder_kl_open_sora_plan_<version>`` (cached)."""
    if version in _LOADED:
        return _LOADED[version]
    C.load_cogvideox_vae()  # the videosys namespace package and the diffusers stand-ins
    cm = C._ensure_mod("diffusers.configuration_utils")
    mm = C._ensure_mod("diffusers.models.modeling_utils")
    C._ensure_mod("diffusers", ConfigMixin=cm.ConfigMixin, ModelMixin=mm.ModelMixin)
    C._ensure_mod("diffusers.utils", logging=types.SimpleNamespace(set_verbosity_error=lambda: None,
                                                                   get_logger=lambda *a, **k: None))
    _LOADED[version] = importlib.import_module(f"videosys.models.autoencoders.autoencoder_kl_open_sora_plan_{version}")
    return _LOADED[version]


def build_osp_vae(version, **cfg):
    """The reference ``CausalVAEModel(**cfg)`` of ``version`` ("v110" / "v120") in eval mode."""
    m = load_osp_vae(version).CausalVAEModel(**cfg)
    assert isinstance(m, nn.Module)
    return m.eval()
