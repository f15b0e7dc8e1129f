"""TEST INFRASTRUCTURE ONLY -- a CPU restatement of the encode path of diffusers' ``AutoencoderKL`` (the SDXL image VAE
that OpenSora v1.2's ``VideoAutoencoderKL.encode`` calls), next to the decode path of oracle/sd_vae_ref.py.

diffusers is not installed here; this file restates, in plain eager torch and with diffusers' parameter names, the facts
of diffusers 0.30's ``AutoencoderKL.encode`` / ``Encoder`` / ``DownEncoderBlock2D`` / ``Downsample2D`` /
``DiagonalGaussianDistribution`` that the encode path uses:
  - ``encoder.conv_in``: 3x3 Conv2d 3 -> block_out_channels[0];
  - ``encoder.down_blocks.{i}`` over block_out_channels: layers_per_block ``resnets`` (ResnetBlock2D, eps 1e-6), the
    first taking the previous block's width; all but the last end in ``downsamplers.0``: Downsample2D with use_conv and
    padding 0, i.e. F.pad(x, (0, 1, 0, 1)) then a 3x3 ``conv`` with stride 2;
  - ``encoder.mid_block``: ``resnets.0``, ``attentions.0``, ``resnets.1`` (as in the decoder);
  - ``encoder.conv_norm_out`` GroupNorm(32, block_out_channels[-1], eps 1e-6), ``conv_act`` SiLU, ``conv_out`` 3x3 ->
    2 * latent_channels (double_z);
  - ``quant_conv``: 1x1 Conv2d 2 * latent -> 2 * latent; ``encode(x).latent_dist`` is
    ``DiagonalGaussianDistribution(moments)``: mean, logvar = chunk(moments, 2, dim=1), logvar clamped to [-30, 20],
    std = exp(0.5 * logvar); ``sample()`` = mean + std * randn_tensor(mean.shape, generator=None,
    device=moments.device, dtype=moments.dtype), randn_tensor being torch.randn on that device.
Slicing and tiling are off (the defaults)."""
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import sd_vae_ref as D


class Downsample2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))


class DownEncoderBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([D.ResnetBlock2D(in_channels if i == 0 else out_channels, out_channels)
                                      for i in range(num_layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(out_channels)]) if add_downsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
        return x


class Encoder(nn.Module):
    def __init__(self, in_channels, latent_channels, block_out_channels, layers_per_block):
        super().__init__()
        self.conv_in = nn.Conv2d(in_channels, block_out_channels[0], 3, padding=1)
        self.down_blocks = nn.ModuleList()
        prev = block_out_channels[0]
        for i, ch in enumerate(block_out_channels):
            self.down_blocks.append(DownEncoderBlock2D(prev, ch, layers_per_block, i < len(block_out_channels) - 1))
            prev = ch
        self.mid_block = D.UNetMidBlock2D(prev)
        self.conv_norm_out = nn.GroupNorm(32, prev, eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(prev, 2 * latent_channels, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for down in self.down_blocks:
            x = down(x)
        return self.conv_out(self.conv_act(self.conv_norm_out(self.mid_block(x))))


class DiagonalGaussianDistribution:
    def __init__(self, parameters):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self):
        noise = torch.randn(self.mean.shape, device=self.parameters.device, dtype=self.parameters.dtype)
        return self.mean + self.std * noise


class AutoencoderKL(D.AutoencoderKL):
    """diffusers' AutoencoderKL, both halves: the decoder of oracle/sd_vae_ref.py plus ``encoder`` and ``quant_conv``;
    ``encode(x).latent_dist`` as diffusers returns it."""

    def __init__(self, block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4):
        super().__init__(block_out_channels, layers_per_block, latent_channels)
        self.encoder = Encoder(3, latent_channels, block_out_channels, layers_per_block)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)

    def encode(self, x):
        return types.SimpleNamespace(latent_dist=DiagonalGaussianDistribution(self.quant_conv(self.encoder(x))))


def build_opensora_vae_full(spatial_block_out_channels=(128, 256, 512, 512), micro_frame_size=17):
    """The reference ``VideoAutoencoderPipeline`` (oracle/opensora_vae_ref.py) with both halves of the image VAE: its
    ``encode`` runs unmodified on this file's AutoencoderKL."""
    from oracle import opensora_vae_ref as R

    m = R.load_opensora_vae()
    bound = m.AutoencoderKL
    m.AutoencoderKL = types.SimpleNamespace(from_pretrained=lambda *a, **k: AutoencoderKL(spatial_block_out_channels))
    try:
        return R.build_opensora_vae(spatial_block_out_channels, micro_frame_size)
    finally:
        m.AutoencoderKL = bound
