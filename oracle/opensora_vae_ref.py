"""TEST INFRASTRUCTURE ONLY -- loads the reference's OpenSora v1.2 VAE (videosys/models/autoencoders/
autoencoder_kl_open_sora.py) unmodified, on the reference checkout that oracle/ref_loader.py finds.

Its imports are einops and transformers (installed) and ``diffusers.models.AutoencoderKL`` /
``AutoencoderKLTemporalDecoder``.  diffusers is not installed: ``AutoencoderKL.from_pretrained`` is a stand-in that returns
the restated decoder of oracle/sd_vae_ref.py (no hub access) with the block widths set by ``build_opensora_vae``.  So the
reference's micro-batching, scale / shift, temporal VAE and ``VideoAutoencoderKL.decode`` run as written; only the body of
diffusers' AutoencoderKL is a restatement.
"""
import importlib

from oracle import cogvideox_vae_ref as C
from oracle import sd_vae_ref

_LOADED = {}
_SPATIAL = {"block_out_channels": (128, 256, 512, 512)}


class _AutoencoderKLStandIn:
    @staticmethod
    def from_pretrained(name, cache_dir=None, local_files_only=False, subfolder=None):
        return sd_vae_ref.AutoencoderKL(_SPATIAL["block_out_channels"])


class _NotAvailable:
    @staticmethod
    def from_pretrained(*a, **k):
        raise NotImplementedError("AutoencoderKLTemporalDecoder has no stand-in")


def load_opensora_vae():
    """The reference module ``videosys.models.autoencoders.autoencoder_kl_open_sora`` (cached)."""
    if "vae" in _LOADED:
        return _LOADED["vae"]
    C.load_cogvideox_vae()  # the videosys namespace package and the diffusers stand-ins
    C._ensure_mod("diffusers.models", AutoencoderKL=_AutoencoderKLStandIn, AutoencoderKLTemporalDecoder=_NotAvailable)
    _LOADED["vae"] = importlib.import_module("videosys.models.autoencoders.autoencoder_kl_open_sora")
    return _LOADED["vae"]


def build_opensora_vae(spatial_block_out_channels=(128, 256, 512, 512), micro_frame_size=17):
    """The reference ``VideoAutoencoderPipeline`` as ``OpenSoraVAE_V1_2`` configures it (:731-761; built from its config
    rather than from a hub checkpoint), with the image decoder's widths given, in eval mode."""
    m = load_opensora_vae()
    cfg = m.VideoAutoencoderPipelineConfig(
        vae_2d=dict(type="VideoAutoencoderKL", from_pretrained="PixArt-alpha/pixart_sigma_sdxlvae_T5_diffusers",
                    subfolder="vae", micro_batch_size=4),
        vae_temporal=dict(type="VAE_Temporal_SD", from_pretrained=None), freeze_vae_2d=False, cal_loss=False,
        micro_frame_size=micro_frame_size, shift=(-0.10, 0.34, 0.27, 0.98), scale=(3.85, 2.32, 2.33, 3.06))
    _SPATIAL["block_out_channels"] = tuple(spatial_block_out_channels)
    return m.VideoAutoencoderPipeline(cfg).eval()
