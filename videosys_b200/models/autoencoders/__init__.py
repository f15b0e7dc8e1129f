"""VAE decoders and the OpenSora v1.2 VAE encoder (videosys/models/autoencoders and the diffusers VAEs the pipelines load): the CogVideoX, Open-Sora-Plan,
OpenSora v1.2, image (AutoencoderKL) and SVD temporal (AutoencoderKLTemporalDecoder) decoders on sm_90a kernels."""
from .autoencoder_kl_cogvideox import AutoencoderKLCogVideoX  # noqa: F401
from .autoencoder_kl_open_sora_plan import CausalVAEModelV110, CausalVAEModelV120  # noqa: F401
from .autoencoder_kl_open_sora import OpenSoraVAEEncoder, VideoAutoencoderPipeline  # noqa: F401
from .autoencoder_kl import AutoencoderKL  # noqa: F401
from .autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder  # noqa: F401
