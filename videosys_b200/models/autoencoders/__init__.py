"""VAE decoders (videosys/models/autoencoders): the CogVideoX decoder on sm_90a kernels."""
from .autoencoder_kl_cogvideox import AutoencoderKLCogVideoX  # noqa: F401
