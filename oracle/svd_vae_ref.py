"""TEST INFRASTRUCTURE ONLY -- a CPU restatement of the decode path of diffusers' ``AutoencoderKLTemporalDecoder`` (the
Stable Video Diffusion VAE that Latte-1 loads from its ``vae_temporal_decoder/`` folder, reference
pipelines/latte/pipeline_latte.py:211-214).

diffusers is not installed here, so the module cannot be imported; this file restates, in plain eager torch on NCHW /
NCDHW tensors, the facts of diffusers 0.30 (models/autoencoders/autoencoder_kl_temporal_decoder.py, unets/
unet_3d_blocks.py ``MidBlockTemporalDecoder`` / ``UpBlockTemporalDecoder``, resnet.py ``SpatioTemporalResBlock`` /
``TemporalResnetBlock`` / ``AlphaBlender``) that the decode path uses, with diffusers' parameter names, reusing the
``ResnetBlock2D`` / ``Attention`` / ``Upsample2D`` leaves of oracle/sd_vae_ref.py:
  - ``decode(z, num_frames)``: no ``post_quant_conv``; z [b * num_frames, C, h, w] is b videos of num_frames frames;
  - ``decoder.conv_in``: 3x3, latent -> block_out_channels[-1];
  - ``decoder.mid_block``: ``resnets.0``, then ``attentions.0``, then ``resnets.1`` (layers_per_block resnets built, the
    forward zips ``resnets[1:]`` with the one attention); the attention is one head of dim C, GroupNorm(32, eps 1e-6),
    biased ``to_q`` / ``to_k`` / ``to_v`` / ``to_out.0``, the residual added;
  - ``decoder.up_blocks.{i}`` over the reversed widths: layers_per_block + 1 resnets each, all but the last ending in
    ``upsamplers.0.conv`` (nearest 2x, then a 3x3 conv);
  - the tail: ``conv_norm_out`` (GroupNorm 32, eps 1e-6) -> SiLU -> ``conv_out`` (3x3 -> 3) -> ``time_conv_out`` (Conv3d
    3 -> 3, kernel (3, 1, 1), padding (1, 0, 0), bias) over (batch, channels, frames, h, w);
  - every resnet is a ``SpatioTemporalResBlock``: ``spatial_res_block`` = ``ResnetBlock2D(in, out)`` (eps 1e-6,
    ``conv_shortcut`` where the width changes, GroupNorm per frame); ``temporal_res_block`` = ``TemporalResnetBlock(out,
    out)``: norm1 -> SiLU -> conv1 -> norm2 -> SiLU -> conv2, + input, both convs (3, 1, 1) with padding (1, 0, 0) and
    bias, GroupNorm(32, eps 1e-5) over C/G x T x H x W of each video, no ``time_emb_proj``; ``time_mixer`` =
    ``AlphaBlender`` (``mix_factor`` [1], merge_strategy "learned", switch_spatial_to_temporal_mix): alpha =
    1 - sigmoid(mix_factor), out = alpha * spatial + (1 - alpha) * temporal.
Only the decoder exists here."""
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.sd_vae_ref import Attention, ResnetBlock2D, Upsample2D


class AlphaBlender(nn.Module):
    def __init__(self, alpha=0.0):
        super().__init__()
        self.mix_factor = nn.Parameter(torch.Tensor([alpha]))

    def forward(self, x_spatial, x_temporal):
        alpha = torch.sigmoid(self.mix_factor).to(x_spatial.dtype)
        alpha = 1.0 - alpha  # switch_spatial_to_temporal_mix
        return alpha * x_spatial + (1.0 - alpha) * x_temporal


class TemporalResnetBlock(nn.Module):
    def __init__(self, in_channels, out_channels, eps=1e-5):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, in_channels, eps=eps)
        self.conv1 = nn.Conv3d(in_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))
        self.norm2 = nn.GroupNorm(32, out_channels, eps=eps)
        self.conv2 = nn.Conv3d(out_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))

    def forward(self, x):
        h = self.conv1(F.silu(self.norm1(x)))
        h = self.conv2(F.silu(self.norm2(h)))
        return x + h


class SpatioTemporalResBlock(nn.Module):
    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.spatial_res_block = ResnetBlock2D(in_channels, out_channels)
        self.temporal_res_block = TemporalResnetBlock(out_channels, out_channels, eps=1e-5)
        self.time_mixer = AlphaBlender()

    def forward(self, x, num_frames):
        x = self.spatial_res_block(x)
        bf, c, h, w = x.shape
        mix = x[None, :].reshape(bf // num_frames, num_frames, c, h, w).permute(0, 2, 1, 3, 4)
        t = self.temporal_res_block(mix)
        x = self.time_mixer(mix, t)
        return x.permute(0, 2, 1, 3, 4).reshape(bf, c, h, w)


class MidBlockTemporalDecoder(nn.Module):
    def __init__(self, channels, num_layers):
        super().__init__()
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(channels, channels) for _ in range(num_layers)])
        self.attentions = nn.ModuleList([Attention(channels)])

    def forward(self, x, num_frames):
        x = self.resnets[0](x, num_frames)
        for resnet, attn in zip(self.resnets[1:], self.attentions):
            x = resnet(attn(x), num_frames)
        return x


class UpBlockTemporalDecoder(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(in_channels if i == 0 else out_channels, out_channels)
                                      for i in range(num_layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(out_channels)]) if add_upsample else None

    def forward(self, x, num_frames):
        for r in self.resnets:
            x = r(x, num_frames)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class TemporalDecoder(nn.Module):
    def __init__(self, in_channels, block_out_channels, layers_per_block):
        super().__init__()
        rev = list(reversed(block_out_channels))
        self.conv_in = nn.Conv2d(in_channels, rev[0], 3, padding=1)
        self.mid_block = MidBlockTemporalDecoder(rev[0], layers_per_block)
        self.up_blocks = nn.ModuleList()
        prev = rev[0]
        for i, ch in enumerate(rev):
            self.up_blocks.append(UpBlockTemporalDecoder(prev, ch, layers_per_block + 1, i < len(rev) - 1))
            prev = ch
        self.conv_norm_out = nn.GroupNorm(32, block_out_channels[0], eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], 3, 3, padding=1)
        self.time_conv_out = nn.Conv3d(3, 3, (3, 1, 1), padding=(1, 0, 0))

    def forward(self, z, num_frames):
        x = self.mid_block(self.conv_in(z), num_frames)
        for up in self.up_blocks:
            x = up(x, num_frames)
        x = self.conv_out(self.conv_act(self.conv_norm_out(x)))
        bf, c, h, w = x.shape
        x = x[None, :].reshape(bf // num_frames, num_frames, c, h, w).permute(0, 2, 1, 3, 4)
        x = self.time_conv_out(x)
        return x.permute(0, 2, 1, 3, 4).reshape(bf, c, h, w)


class AutoencoderKLTemporalDecoder(nn.Module):
    """decoder half of diffusers' AutoencoderKLTemporalDecoder; ``decode(z, num_frames).sample`` as diffusers returns it."""

    def __init__(self, block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4, scaling_factor=0.18215):
        super().__init__()
        self.config = types.SimpleNamespace(block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                            latent_channels=latent_channels, scaling_factor=scaling_factor)
        self.decoder = TemporalDecoder(latent_channels, block_out_channels, layers_per_block)

    def decode(self, z, num_frames):
        return types.SimpleNamespace(sample=self.decoder(z, num_frames))
