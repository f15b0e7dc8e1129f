"""diffusers' ``AutoencoderKLTemporalDecoder`` (the Stable Video Diffusion VAE; Latte-1's ``vae_temporal_decoder``),
decoder half, on the sm_90a kernels of csrc/vae_conv.cu, with diffusers' parameter names under ``decoder.*``.

The facts restated here (diffusers 0.30: models/autoencoders/autoencoder_kl_temporal_decoder.py, unets/unet_3d_blocks.py
``MidBlockTemporalDecoder`` / ``UpBlockTemporalDecoder``, resnet.py ``SpatioTemporalResBlock`` / ``TemporalResnetBlock`` /
``AlphaBlender``):
  - ``decode(z, num_frames)``: no ``post_quant_conv``; z [b * num_frames, C, h, w] is b videos of num_frames frames.
  - ``decoder.conv_in``: 3x3, latent -> block_out_channels[-1].
  - ``decoder.mid_block``: ``resnets.0``, then ``attentions.0``, then ``resnets.1`` (layers_per_block resnets are built;
    the forward pairs ``resnets[1:]`` with the one attention).  The attention is one head of dim C, GroupNorm(32, eps
    1e-6), biased ``to_q`` / ``to_k`` / ``to_v`` / ``to_out.0``, the residual added.
  - ``decoder.up_blocks.{i}`` over the reversed widths: layers_per_block + 1 resnets each; all but the last end in
    ``upsamplers.0.conv`` (nearest 2x, then a 3x3 conv).
  - The tail: ``conv_norm_out`` (GroupNorm 32, eps 1e-6) -> SiLU -> ``conv_out`` (3x3 -> 3) -> ``time_conv_out`` (Conv3d
    3 -> 3, kernel (3, 1, 1), padding (1, 0, 0), bias) over each video's frames.
  - Every resnet is a ``SpatioTemporalResBlock``:
      ``spatial_res_block`` = ``ResnetBlock2D(in, out)``, eps 1e-6, ``conv_shortcut`` where the width changes, GroupNorm
      per frame;
      ``temporal_res_block`` = ``TemporalResnetBlock(out, out)``: norm1 -> SiLU -> conv1 -> norm2 -> SiLU -> conv2, + its
      input; both convs (3, 1, 1) with padding (1, 0, 0) and bias; GroupNorm(32, eps 1e-5) over C/G x T x H x W of each
      video (not per frame); no ``time_emb_proj``;
      ``time_mixer`` = ``AlphaBlender``: ``mix_factor`` [1], merge_strategy "learned", switch_spatial_to_temporal_mix:
      alpha = 1 - sigmoid(mix_factor), out = alpha * spatial + (1 - alpha) * temporal.
  - ``load_state_dict`` drops ``encoder.*`` and ``quant_conv.*``.

Activations are channels-last: the spatial half sees ``[b * T, 1, H, W, C]`` (each frame its own GroupNorm sample) and
the temporal half the same storage as ``[b, T, H, W, C]``.  The temporal convolutions read a buffer ``[b, T + 2, H, W,
C]`` whose frames 0 and T + 1 are zero (the padding) and whose frames 1 .. T the GroupNorm + SiLU kernel wrote;
``conv2`` carries the TemporalResnetBlock's residual and the AlphaBlender in its epilogue (``vae_conv_time`` with mix).
"""
from typing import Sequence

import torch
import torch.nn as nn

from ... import kernels
from ._common import DecoderOnlyVAE, check_widths, group_norm, pad_latent, run_conv
from .autoencoder_kl import _SILU, Attention, DecoderOutput, ResnetBlock2D, Upsample2D


class AlphaBlender(nn.Module):
    """merge_strategy "learned", switch_spatial_to_temporal_mix: the blend weights of the spatial and the temporal
    output, computed in the parameter dtype as diffusers computes them (each op rounded)."""

    def __init__(self, alpha: float = 0.0):
        super().__init__()
        self.mix_factor = nn.Parameter(torch.tensor([alpha]))
        self._ab = None

    def pack(self):
        with torch.no_grad():
            a = 1.0 - torch.sigmoid(self.mix_factor)
            b = 1.0 - a
        self._ab = (float(a), float(b))


class TemporalResnetBlock(nn.Module):
    def __init__(self, in_channels, out_channels, eps=1e-5):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, in_channels, eps=eps)
        self.conv1 = nn.Conv3d(in_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))
        self.norm2 = nn.GroupNorm(32, out_channels, eps=eps)
        self.conv2 = nn.Conv3d(out_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))

    def forward(self, x, mix):
        """x [b, T, H, W, C] -> mix[0] * x + mix[1] * (x + block(x))."""
        b, T, H, W, C = x.shape
        buf = torch.empty(b, T + 2, H, W, C, dtype=x.dtype, device=x.device)
        buf[:, 0].zero_()
        buf[:, T + 1].zero_()
        group_norm(self.norm1, x, buf, t_off=1, act=_SILU)
        h = kernels.vae_conv_time(buf, self.conv1._w, self.conv1._b, C, 3)
        group_norm(self.norm2, h, buf, t_off=1, act=_SILU)  # conv1 has read buf: same stream
        return kernels.vae_conv_time(buf, self.conv2._w, self.conv2._b, C, 3, resid=x, mix=mix)


class SpatioTemporalResBlock(nn.Module):
    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.spatial_res_block = ResnetBlock2D(in_channels, out_channels, eps=1e-6)
        self.temporal_res_block = TemporalResnetBlock(out_channels, out_channels, eps=1e-5)
        self.time_mixer = AlphaBlender()

    def forward(self, x, num_frames):
        """x [b * T, 1, H, W, Cin] -> [b * T, 1, H, W, Cout]."""
        xs = self.spatial_res_block(x)
        N, _, H, W, C = xs.shape
        out = self.temporal_res_block(xs.view(N // num_frames, num_frames, H, W, C), self.time_mixer._ab)
        return out.view(N, 1, H, W, C)


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
    def __init__(self, in_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2):
        super().__init__()
        rev = list(reversed(block_out_channels))
        self.conv_in = nn.Conv2d(in_channels, rev[0], 3, padding=1)
        self.mid_block = MidBlockTemporalDecoder(rev[0], layers_per_block)
        self.up_blocks = nn.ModuleList([])
        prev = rev[0]
        for i, ch in enumerate(rev):
            self.up_blocks.append(UpBlockTemporalDecoder(prev, ch, layers_per_block + 1, add_upsample=i < len(rev) - 1))
            prev = ch
        self.conv_norm_out = nn.GroupNorm(32, block_out_channels[0], eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], out_channels, 3, padding=1)
        self.time_conv_out = nn.Conv3d(out_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))

    def forward(self, z, num_frames):
        """z [b * T, 1, h, w, 16] (zero padded) -> [b * T, 1, 8h, 8w, 3]."""
        x = self.mid_block(run_conv(self.conv_in, z), num_frames)
        for up in self.up_blocks:
            x = up(x, num_frames)
        x = run_conv(self.conv_out, group_norm(self.conv_norm_out, x, act=_SILU))
        N, _, H, W, C = x.shape
        v = kernels.vae_time_conv_rgb(x.view(N // num_frames, num_frames, H, W, C), self.time_conv_out.weight,
                                      self.time_conv_out.bias)
        return v.view(N, 1, H, W, C)


class AutoencoderKLTemporalDecoder(DecoderOnlyVAE):
    """diffusers' AutoencoderKLTemporalDecoder, decoder only (see the module docstring).  Stable Video Diffusion's and
    Latte-1's have block_out_channels (128, 256, 512, 512), layers_per_block 2, latent_channels 4."""

    _DROPPED_PREFIXES = ("encoder.", "quant_conv.")

    def __init__(self, in_channels: int = 3, out_channels: int = 3,
                 block_out_channels: Sequence[int] = (128, 256, 512, 512), layers_per_block: int = 2,
                 latent_channels: int = 4, sample_size: int = 32, scaling_factor: float = 0.18215,
                 force_upcast: float = True):
        super().__init__()
        if out_channels != 3:
            raise NotImplementedError(f"out_channels={out_channels}: time_conv_out runs on RGB")
        if not 1 <= latent_channels <= 16:
            raise NotImplementedError(f"latent_channels={latent_channels}: the latent is padded to 16 channels")
        check_widths(block_out_channels, f"block_out_channels={tuple(block_out_channels)}")
        self.config = type("Config", (), dict(
            in_channels=in_channels, out_channels=out_channels, block_out_channels=tuple(block_out_channels),
            layers_per_block=layers_per_block, latent_channels=latent_channels, sample_size=sample_size,
            scaling_factor=scaling_factor, force_upcast=force_upcast))()
        self.decoder = TemporalDecoder(latent_channels, out_channels, tuple(block_out_channels), layers_per_block)

    @classmethod
    def from_pretrained(cls, path: str, subfolder: str = "vae_temporal_decoder"):
        """A LOCAL diffusers snapshot (``<path>/<subfolder>/config.json`` + weights); no hub download."""
        return cls._from_local_diffusers(path, subfolder)

    @property
    def dtype(self):
        return self.decoder.conv_in.weight.dtype

    @property
    def device(self):
        return self.decoder.conv_in.weight.device

    @torch.no_grad()
    def decode(self, z, num_frames: int, return_dict: bool = True):
        """z [b * num_frames, latent_channels, h, w] -> ``.sample`` [b * num_frames, 3, 8h, 8w]."""
        if z.shape[0] % num_frames:
            raise ValueError(f"decode: {z.shape[0]} frames are not whole videos of num_frames={num_frames}")
        z = self._decode_input(z)
        x = self.decoder(pad_latent(z.permute(0, 2, 3, 1))[:, None], num_frames)
        dec = x[:, 0].permute(0, 3, 1, 2)
        return DecoderOutput(sample=dec) if return_dict else (dec,)
