"""VAE decoders (videosys/models/autoencoders): the CogVideoX, Open-Sora-Plan and OpenSora v1.2 decoders on sm_90a kernels."""
from .autoencoder_kl_cogvideox import AutoencoderKLCogVideoX  # noqa: F401
from .autoencoder_kl_open_sora_plan import CausalVAEModelV110, CausalVAEModelV120  # noqa: F401
from .autoencoder_kl_open_sora import VideoAutoencoderPipeline  # noqa: F401
