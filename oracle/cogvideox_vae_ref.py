"""TEST INFRASTRUCTURE ONLY -- loads the reference's CogVideoX VAE (videosys/models/autoencoders/autoencoder_kl_cogvideox.py
and videosys/models/modules/upsampling.py) unmodified, on the reference checkout that oracle/ref_loader.py finds.

Its diffusers imports (:18-24) are mixins and output containers; they are replaced by the stand-ins below.  The only
arithmetic among them is ``get_activation("silu")``, which maps to ``nn.SiLU``.  ``register_to_config`` records the
constructor's keywords in ``self.config`` before the constructor body runs, as diffusers does.
"""
import functools
import importlib
import inspect
import sys
import types

import torch.nn as nn

from oracle import ref_loader

_LOADED = {}


def _ensure_mod(name, **kw):
    m = sys.modules.get(name)
    if m is None:
        m = types.ModuleType(name)
        sys.modules[name] = m
    m.__dict__.update(kw)
    return m


def _register_to_config(init):
    @functools.wraps(init)
    def wrapped(self, *args, **kwargs):
        bound = inspect.signature(init).bind(self, *args, **kwargs)
        bound.apply_defaults()
        cfg = {k: v for k, v in bound.arguments.items() if k != "self"}
        object.__setattr__(self, "config", types.SimpleNamespace(**cfg))
        init(self, *args, **kwargs)

    return wrapped


class _Output:
    def __init__(self, sample=None, **kw):
        self.sample = sample
        self.__dict__.update(kw)


def _get_activation(name):
    if name in ("silu", "swish"):
        return nn.SiLU()
    raise ValueError(f"activation {name!r} has no stand-in")


def load_cogvideox_vae():
    """The reference module ``videosys.models.autoencoders.autoencoder_kl_cogvideox`` (cached)."""
    if _LOADED:
        return _LOADED["vae"]
    if not ref_loader.available():
        raise RuntimeError(f"reference tree not present at {ref_loader.REF}")
    if "videosys" not in sys.modules:
        pkg = _ensure_mod("videosys")
        pkg.__path__ = [ref_loader.REF + "/videosys"]
    _ensure_mod("diffusers")
    _ensure_mod("diffusers.configuration_utils", ConfigMixin=type("ConfigMixin", (), {}), register_to_config=_register_to_config)
    _ensure_mod("diffusers.loaders")
    _ensure_mod("diffusers.loaders.single_file_model", FromOriginalModelMixin=type("FromOriginalModelMixin", (), {}))
    _ensure_mod("diffusers.models")
    _ensure_mod("diffusers.models.activations", get_activation=_get_activation)
    _ensure_mod("diffusers.models.autoencoders")
    _ensure_mod("diffusers.models.autoencoders.vae", DecoderOutput=_Output, DiagonalGaussianDistribution=_Output)
    _ensure_mod("diffusers.models.modeling_outputs", AutoencoderKLOutput=_Output)
    _ensure_mod("diffusers.models.modeling_utils", ModelMixin=nn.Module)
    _ensure_mod("diffusers.utils")
    _ensure_mod("diffusers.utils.accelerate_utils", apply_forward_hook=lambda f: f)
    _LOADED["vae"] = importlib.import_module("videosys.models.autoencoders.autoencoder_kl_cogvideox")
    return _LOADED["vae"]


def build_cogvideox_vae(**cfg):
    """The reference ``AutoencoderKLCogVideoX(**cfg)`` in eval mode."""
    return load_cogvideox_vae().AutoencoderKLCogVideoX(**cfg).eval()
