"""OpenSora v1.2 VAE decoder and encoder (mirror of videosys/models/autoencoders/autoencoder_kl_open_sora.py:
DiagonalGaussianDistribution :21-64, CausalConv3d :89-124, ResBlock :127-164, Encoder :177-272, Decoder :275-376, VAE_Temporal :379-471, VAE_Temporal_SD :474-485, VideoAutoencoderKL :488-555,
VideoAutoencoderPipeline :621-729) on the sm_90a kernels of csrc/vae_conv.cu and csrc/vae_osp.cu.

``VideoAutoencoderPipeline`` is the decoder half (its ``encode`` raises ``NotImplementedError``); ``OpenSoraVAEEncoder``
is the encoder half of the same checkpoint (see its docstring).  ``decode(z, num_frames)`` runs the reference's three
stages:
  1. ``z * scale + shift`` (persistent buffers, so a checkpoint's values load over the released ones);
  2. the temporal decoder (``temporal_vae``) per micro-batch of ``micro_z_frame_size`` = 5 latent frames, each chunk on its
     own (no causal state between chunks), with its leading ``time_padding`` frames trimmed;
  3. the SDXL image decoder (``spatial_vae.module``, diffusers' ``AutoencoderKL`` of autoencoder_kl.py: diffusers'
     parameter names) on ``micro_batch_size`` frames at a time, each frame its own GroupNorm sample, after ``x / 0.18215``.
Activations stay channels-last ``[B, T, H, W, C]`` between kernels:
  - every temporal causal convolution reads a buffer whose kt - 1 = 2 leading context frames are ZEROS (the reference
    pads with ``F.pad(mode="constant")``), followed by the frames the previous kernel wrote there (GroupNorm + SiLU);
  - the image decoder holds its frames in the batch dimension with T = 1, and its 3x3 convolutions are kt = 1;
  - the 4-channel latent is zero padded to 16 channels; ``post_quant_conv`` (both stages) and the 1x1 shortcuts are GEMMs
    on the pixel rows;
  - the depth-to-time shuffle after each temporal up-sampling conv (``rearrange("B (C ts) T H W -> B C (T ts) H W")``) is
    ``vae_depth_to_time``;
  - the image decoder's mid-block attention runs q | k | v as one GEMM, S = Q K^T, the scaled softmax and O = P V per
    frame (materialised), and ``to_out`` with the residual in the GEMM epilogue.
Every nonlinearity is ``nn.SiLU`` (``vae_groupnorm_act(act=2)``: one fp32 evaluation, one rounding).
"""
import os
from typing import Optional, Sequence

import torch
import torch.nn as nn

from ... import kernels
from ._common import (LATENT_PAD, DecoderOnlyVAE, _cast_tuple, check_widths, conv_buffer, conv_kt, group_norm, pad_1x1,
                      pad_latent, run_conv)
from .autoencoder_kl import _SILU, AutoencoderKL, SpatialEncoder
SCALE = (3.85, 2.32, 2.33, 3.06)  # OpenSoraVAE_V1_2 (:748-749)
SHIFT = (-0.10, 0.34, 0.27, 0.98)
SD_SCALING = 0.18215  # VideoAutoencoderKL.decode divides the latent by this (:534)


# =====================================================================================================================
# temporal decoder (VAE_Temporal_SD)
# =====================================================================================================================
class CausalConv3d(nn.Module):
    """Reference :89-124: kt - 1 leading ZERO frames, zero spatial padding, then nn.Conv3d (``conv.*``)."""

    def __init__(self, chan_in, chan_out, kernel_size, bias=True):
        super().__init__()
        self.conv = nn.Conv3d(chan_in, chan_out, _cast_tuple(kernel_size, 3), bias=bias)

    def input_buffer(self, x_shape, dtype, device):
        """conv_buffer with the kt - 1 context frames zeroed."""
        buf = conv_buffer(self.conv, x_shape, dtype, device)
        buf[:, :conv_kt(self.conv) - 1].zero_()
        return buf

    def run(self, buf, resid=None):
        return run_conv(self.conv, buf, resid)


class ResBlock(nn.Module):
    """Reference :127-164: norm1 -> SiLU -> conv1 -> norm2 -> SiLU -> conv2, + x (through the bias-free 1x1x1 conv3 when
    the width changes) in conv2's epilogue.  GroupNorm eps is torch's default 1e-5."""

    def __init__(self, in_channels, filters, num_groups=32):
        super().__init__()
        self.in_channels, self.filters = in_channels, filters
        self.norm1 = nn.GroupNorm(num_groups, in_channels)
        self.conv1 = CausalConv3d(in_channels, filters, (3, 3, 3), bias=False)
        self.norm2 = nn.GroupNorm(num_groups, filters)
        self.conv2 = CausalConv3d(filters, filters, (3, 3, 3), bias=False)
        if in_channels != filters:
            self.conv3 = CausalConv3d(in_channels, filters, (1, 1, 1), bias=False)

    def forward(self, x):
        buf = self.conv1.input_buffer(x.shape, x.dtype, x.device)
        group_norm(self.norm1, x, buf, t_off=2, act=_SILU)
        h = self.conv1.run(buf)
        buf = self.conv2.input_buffer(h.shape, h.dtype, h.device)
        group_norm(self.norm2, h, buf, t_off=2, act=_SILU)
        if self.in_channels != self.filters:
            x = kernels.gemm_bias_act(x, self.conv3.conv._w)
        return self.conv2.run(buf, resid=x)


class Decoder(nn.Module):
    """Reference :275-376: conv1, num_res_blocks ResBlocks, then per level (widest first) num_res_blocks ResBlocks and,
    where temporal_downsample[i - 1] is set, a 3x3x3 conv to twice the width and the depth-to-time shuffle; norm1 + SiLU,
    conv_out.  Levels without a temporal up-sampling keep an ``nn.Identity`` in ``conv_blocks`` (no parameters)."""

    def __init__(self, in_out_channels=4, latent_embed_dim=512, filters=128, num_res_blocks=4,
                 channel_multipliers=(1, 2, 2, 4), temporal_downsample=(False, True, True), num_groups=32):
        super().__init__()
        self.num_res_blocks = num_res_blocks
        self.num_blocks = len(channel_multipliers)
        self.temporal_downsample = temporal_downsample
        filters_ = filters * channel_multipliers[-1]
        prev = filters_
        self.conv1 = CausalConv3d(latent_embed_dim, filters_, (3, 3, 3), bias=True)
        self.res_blocks = nn.ModuleList([ResBlock(filters_, filters_, num_groups) for _ in range(num_res_blocks)])
        self.block_res_blocks = nn.ModuleList([])
        self.conv_blocks = nn.ModuleList([])
        for i in reversed(range(self.num_blocks)):
            filters_ = filters * channel_multipliers[i]
            items = nn.ModuleList([])
            for _ in range(num_res_blocks):
                items.append(ResBlock(prev, filters_, num_groups))
                prev = filters_
            self.block_res_blocks.insert(0, items)
            if i > 0:
                self.conv_blocks.insert(0, CausalConv3d(prev, prev * 2, (3, 3, 3)) if temporal_downsample[i - 1] else nn.Identity())
        self.norm1 = nn.GroupNorm(num_groups, prev)
        self.conv_out = CausalConv3d(filters_, in_out_channels, 3)

    def forward(self, z):
        """z [B, T, h, w, 16] (channels-last, zero padded) -> [B, 4 T', h, w, in_out_channels], T' = T * 2^(up-samplings)."""
        buf = self.conv1.input_buffer(z.shape, z.dtype, z.device)
        buf[:, 2:] = z
        x = self.conv1.run(buf)
        for b in self.res_blocks:
            x = b(x)
        for i in reversed(range(self.num_blocks)):
            for b in self.block_res_blocks[i]:
                x = b(x)
            if i > 0 and self.temporal_downsample[i - 1]:
                conv = self.conv_blocks[i - 1]
                buf = conv.input_buffer(x.shape, x.dtype, x.device)
                buf[:, 2:] = x
                x = kernels.vae_depth_to_time(conv.run(buf))
        buf = self.conv_out.input_buffer(x.shape, x.dtype, x.device)
        group_norm(self.norm1, x, buf, t_off=2, act=_SILU)
        return self.conv_out.run(buf)


class VAE_Temporal(nn.Module):
    """Reference :379-471, decoder half: ``post_quant_conv`` (1x1x1, bias) and ``decoder``."""

    def __init__(self, in_out_channels=4, latent_embed_dim=4, embed_dim=4, filters=128, num_res_blocks=4,
                 channel_multipliers=(1, 2, 2, 4), temporal_downsample=(True, True, False), num_groups=32):
        super().__init__()
        self.time_downsample_factor = 2 ** sum(temporal_downsample)
        self.patch_size = (self.time_downsample_factor, 1, 1)
        self.out_channels = in_out_channels
        self.post_quant_conv = CausalConv3d(embed_dim, latent_embed_dim, 1)
        self.decoder = Decoder(in_out_channels=in_out_channels, latent_embed_dim=latent_embed_dim, filters=filters,
                               num_res_blocks=num_res_blocks, channel_multipliers=channel_multipliers,
                               temporal_downsample=temporal_downsample, num_groups=num_groups)
        self._pq = None

    def pack(self):
        self._pq = pad_1x1(self.post_quant_conv.conv.weight, self.post_quant_conv.conv.bias)

    def get_latent_size(self, input_size):
        """Reference :424-439."""
        out = []
        for i in range(3):
            if input_size[i] is None:
                out.append(None)
            elif i == 0:
                pad = 0 if input_size[i] % self.time_downsample_factor == 0 else \
                    self.time_downsample_factor - input_size[i] % self.time_downsample_factor
                out.append((input_size[i] + pad) // self.patch_size[i])
            else:
                out.append(input_size[i] // self.patch_size[i])
        return out

    def decode(self, z, num_frames):
        """z [B, T, h, w, 16] channels-last -> [B, 4T - time_padding, h, w, 4] (reference :453-462)."""
        pad = 0 if num_frames % self.time_downsample_factor == 0 else \
            self.time_downsample_factor - num_frames % self.time_downsample_factor
        x = self.decoder(kernels.gemm_bias_act(z, *self._pq))
        return x[:, pad:]


def VAE_Temporal_SD(**kwargs):
    """Reference :474-485: the released temporal VAE."""
    return VAE_Temporal(in_out_channels=4, latent_embed_dim=4, embed_dim=4, filters=128, num_res_blocks=4,
                        channel_multipliers=(1, 2, 2, 4), temporal_downsample=(False, True, True), **kwargs)


class VideoAutoencoderKL(nn.Module):
    """Reference :488-555, decoder half: frames folded into the batch, ``micro_batch_size`` at a time."""

    def __init__(self, micro_batch_size: Optional[int] = 4, block_out_channels: Sequence[int] = (128, 256, 512, 512)):
        super().__init__()
        self.module = AutoencoderKL(block_out_channels=block_out_channels)
        self.out_channels = self.module.config.latent_channels
        self.patch_size = (1, 8, 8)
        self.micro_batch_size = micro_batch_size

    def decode(self, x):
        """x [B, T, h, w, 4] channels-last -> [B, T, 8h, 8w, 3] (reference :522-538)."""
        B, T, h, w, C = x.shape
        x = x.reshape(B * T, 1, h, w, C)
        N = B * T
        bs = N if self.micro_batch_size is None else self.micro_batch_size
        out = torch.empty(N, 1, 8 * h, 8 * w, 3, dtype=x.dtype, device=x.device)
        for i in range(0, N, bs):
            out[i:i + bs] = self.module.decode_frames(pad_latent(x[i:i + bs] / SD_SCALING))
        return out.view(B, T, 8 * h, 8 * w, 3)


# =====================================================================================================================
# the pipeline
# =====================================================================================================================
class VideoAutoencoderPipeline(DecoderOnlyVAE):
    """OpenSora v1.2 VAE (reference :621-729 as built by OpenSoraVAE_V1_2 :731-761), decoder only: ``temporal_vae``
    (VAE_Temporal_SD) and ``spatial_vae.module`` (the SDXL AutoencoderKL), ``scale`` / ``shift`` buffers.

    ``spatial_block_out_channels`` narrows the image decoder (tests); every width must be one the GroupNorm kernels take
    (64, 128, 256, 512).  ``load_state_dict`` takes the checkpoint's full state dict: it drops ``*.encoder.*`` and
    ``*.quant_conv.*`` and is strict about every other key (``scale`` / ``shift`` may be absent: the released values stay).
    """

    def __init__(self, micro_frame_size: Optional[int] = 17, micro_batch_size: Optional[int] = 4,
                 spatial_block_out_channels: Sequence[int] = (128, 256, 512, 512), scale=SCALE, shift=SHIFT):
        super().__init__()
        check_widths(spatial_block_out_channels, f"spatial_block_out_channels={tuple(spatial_block_out_channels)}")
        self.spatial_vae = VideoAutoencoderKL(micro_batch_size, spatial_block_out_channels)
        self.temporal_vae = VAE_Temporal_SD()
        self.micro_frame_size = micro_frame_size
        self.micro_z_frame_size = self.temporal_vae.get_latent_size([micro_frame_size, None, None])[0] \
            if micro_frame_size is not None else None
        self.out_channels = self.temporal_vae.out_channels
        self.register_buffer("scale", torch.tensor(scale)[None, :, None, None, None])
        self.register_buffer("shift", torch.tensor(shift)[None, :, None, None, None])

    # ---- loading ----
    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, **kwargs):
        """A LOCAL snapshot of hpcai-tech/OpenSora-VAE-v1.2 (``model.safetensors`` and friends, read by
        utils/checkpoint.py).  No hub access."""
        from ...utils.checkpoint import load_local_checkpoint

        _, sd = load_local_checkpoint(path, subfolder or "")
        vae = cls(**kwargs)
        vae.load_state_dict(sd)
        return vae

    def _dropped(self, key: str) -> bool:
        """Encoder-side keys of the full checkpoint (``*.encoder.*``, ``*.quant_conv.*``): not part of the decoder."""
        parts = key.split(".")
        return "encoder" in parts or "quant_conv" in parts

    def load_state_dict(self, state_dict, strict: bool = True):
        defaults = {k: getattr(self, k) for k in ("scale", "shift") if k not in state_dict}
        return super().load_state_dict({**state_dict, **defaults}, strict=strict)

    @property
    def dtype(self):
        return self.temporal_vae.decoder.norm1.weight.dtype

    @property
    def device(self):
        return self.temporal_vae.decoder.norm1.weight.device

    # ---- decoding ----
    @torch.no_grad()
    def decode(self, z, num_frames=None):
        """z [B, 4, T, h, w] -> video [B, 3, T', 8h, 8w] in [-1, 1]-ish (reference decode :672-695, cal_loss off)."""
        z = self._decode_input(z)
        z = z * self.scale.to(z.dtype) + self.shift.to(z.dtype)
        zl = z.permute(0, 2, 3, 4, 1)  # [B, T, h, w, 4]
        if self.micro_frame_size is None:
            x_z = self.temporal_vae.decode(pad_latent(zl), num_frames=num_frames)
        else:
            chunks = []
            for i in range(0, zl.shape[1], self.micro_z_frame_size):
                z_bs = pad_latent(zl[:, i:i + self.micro_z_frame_size])
                chunks.append(self.temporal_vae.decode(z_bs, num_frames=min(self.micro_frame_size, num_frames)))
                num_frames -= self.micro_frame_size
            x_z = torch.cat(chunks, dim=1)
        return self.spatial_vae.decode(x_z).permute(0, 4, 1, 2, 3)


# =====================================================================================================================
# the encoder
# =====================================================================================================================
def _pad_rows(weight, bias, rows=LATENT_PAD):
    """A c' x Cin 1x1 convolution (c' <= 16) as a [16, Cin] GEMM weight and a [16] bias (zero rows)."""
    w = torch.zeros(rows, weight.shape[1], dtype=weight.dtype, device=weight.device)
    w[:weight.shape[0]] = weight.detach().flatten(1)
    b = torch.zeros(rows, dtype=weight.dtype, device=weight.device)
    b[:weight.shape[0]] = bias.detach()
    return w, b


class Encoder(nn.Module):
    """Reference :177-272: conv_in (bias-free), per level num_res_blocks ResBlocks and, between levels, a causal 3x3x3
    conv with stride (2, 1, 1) where temporal_downsample[i] is set (``nn.Identity`` otherwise, no parameters),
    num_res_blocks ResBlocks, norm1 + SiLU, the 1x1x1 conv2 to latent_embed_dim channels."""

    def __init__(self, in_out_channels=4, latent_embed_dim=8, filters=128, num_res_blocks=4,
                 channel_multipliers=(1, 2, 2, 4), temporal_downsample=(False, True, True), num_groups=32):
        super().__init__()
        self.num_blocks = len(channel_multipliers)
        self.temporal_downsample = temporal_downsample
        self.conv_in = CausalConv3d(in_out_channels, filters, (3, 3, 3), bias=False)
        self.block_res_blocks = nn.ModuleList([])
        self.conv_blocks = nn.ModuleList([])
        prev = filters
        for i in range(self.num_blocks):
            filters_ = filters * channel_multipliers[i]
            items = nn.ModuleList([])
            for _ in range(num_res_blocks):
                items.append(ResBlock(prev, filters_, num_groups))
                prev = filters_
            self.block_res_blocks.append(items)
            if i < self.num_blocks - 1:
                self.conv_blocks.append(CausalConv3d(prev, filters_, (3, 3, 3)) if temporal_downsample[i] else nn.Identity())
                prev = filters_
        self.res_blocks = nn.ModuleList([ResBlock(prev, filters_, num_groups) for _ in range(num_res_blocks)])
        self.norm1 = nn.GroupNorm(num_groups, prev)
        self.conv2 = CausalConv3d(prev, latent_embed_dim, 1)
        self._c2 = None

    def pack(self):
        self._c2 = _pad_rows(self.conv2.conv.weight, self.conv2.conv.bias)

    def forward(self, buf):
        """buf [B, 2 + T, h, w, 16]: the conv_in input after its two zero context frames (the latent zero padded to 16
        channels, T a multiple of 4) -> [B, T / 4, h, w, 16], channels latent_embed_dim.. zero."""
        x = self.conv_in.run(buf)
        for i in range(self.num_blocks):
            for b in self.block_res_blocks[i]:
                x = b(x)
            if i < self.num_blocks - 1 and self.temporal_downsample[i]:
                # time_pad = 2 + (1 - 2) = 1 zero frame in front (:110): the kernel's out-of-bounds fill, no copy
                conv = self.conv_blocks[i].conv
                x = kernels.vae_conv_down(x, conv._w, conv._b, conv.out_channels, 3)
        for b in self.res_blocks:
            x = b(x)
        return kernels.gemm_bias_act(group_norm(self.norm1, x, act=_SILU), *self._c2)


class VAE_TemporalEncoder(nn.Module):
    """Reference VAE_Temporal (:379-451), encoder half of VAE_Temporal_SD: ``encoder`` and ``quant_conv`` (1x1x1)."""

    def __init__(self, in_out_channels=4, latent_embed_dim=4, embed_dim=4, filters=128, num_res_blocks=4,
                 channel_multipliers=(1, 2, 2, 4), temporal_downsample=(False, True, True), num_groups=32):
        super().__init__()
        self.time_downsample_factor = 2 ** sum(temporal_downsample)
        self.encoder = Encoder(in_out_channels, 2 * latent_embed_dim, filters, num_res_blocks, channel_multipliers,
                               temporal_downsample, num_groups)
        self.quant_conv = CausalConv3d(2 * latent_embed_dim, 2 * embed_dim, 1)
        self._q = None

    def pack(self):
        self._q = pad_1x1(self.quant_conv.conv.weight, self.quant_conv.conv.bias)

    def moments(self, x):
        """x [B, T, h, w, 4] channels-last -> moments [B, T', h, w, 16] (channels 8.. zero): T front-padded with zero
        frames to a multiple of 4 (:441-449), the encoder, quant_conv."""
        B, T, h, w, c = x.shape
        pad = -T % self.time_downsample_factor
        buf = torch.zeros(B, 2 + pad + T, h, w, LATENT_PAD, dtype=x.dtype, device=x.device)
        buf[:, 2 + pad:, ..., :c] = x
        return kernels.gemm_bias_act(self.encoder(buf), *self._q)


class _ImageEncoder(nn.Module):
    """diffusers' AutoencoderKL, encoder half: ``encoder`` (SpatialEncoder) and ``quant_conv`` (1x1, 8 -> 8)."""

    def __init__(self, block_out_channels):
        super().__init__()
        self.encoder = SpatialEncoder(3, 4, block_out_channels)
        self.quant_conv = nn.Conv2d(8, 8, 1)
        self._q = None

    def pack(self):
        self._q = pad_1x1(self.quant_conv.weight, self.quant_conv.bias)

    def moments(self, x):
        """x [N, 1, H, W, 16] (RGB zero padded) -> moments [N, 1, h, w, 16] (channels 8.. zero)."""
        return kernels.gemm_bias_act(pad_latent(self.encoder(x)), *self._q)


class _SpatialEncoderHolder(nn.Module):
    """Holds the image encoder as ``module`` (the reference's VideoAutoencoderKL.module)."""

    def __init__(self, micro_batch_size, block_out_channels):
        super().__init__()
        self.module = _ImageEncoder(block_out_channels)
        self.micro_batch_size = micro_batch_size


def _sample(moments, noise):
    """DiagonalGaussianDistribution(moments).sample() (:21-39; diffusers' vae.py likewise) on the channels-last moments,
    as the same eager 16-bit ops: mean, logvar = chunk(2), logvar.clamp(-30, 20), std = exp(0.5 * logvar),
    mean + std * noise."""
    mean, logvar = moments[..., :4], moments[..., 4:8]
    std = torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0))
    return mean + std * noise


class OpenSoraVAEEncoder(DecoderOnlyVAE):
    """OpenSora v1.2 VAE, encoder half (reference VideoAutoencoderPipeline.encode :653-670 with cal_loss off):
    ``spatial_vae.module`` (diffusers' AutoencoderKL encoder + quant_conv, the SDXL VAE) and ``temporal_vae``
    (VAE_Temporal_SD's encoder + quant_conv), with the reference's key names.  A module of its own: the decoder
    (VideoAutoencoderPipeline) keeps the decoder half of the same checkpoint.

    ``load_state_dict`` takes the checkpoint's full state dict: it drops the decoder-side keys and is strict about the
    encoder side; ``scale`` / ``shift``, when present, load over the released values (non-persistent buffers).
    ``spatial_block_out_channels`` narrows the image encoder (tests).

    It shares DecoderOnlyVAE's weight packing, config and loading filter, with two overrides: ``_dropped`` is inverted
    (it keeps the encoder prefixes and drops everything else, the decoder side included), and ``encode`` is real."""

    _KEPT_PREFIXES = ("temporal_vae.encoder.", "temporal_vae.quant_conv.", "spatial_vae.module.encoder.",
                      "spatial_vae.module.quant_conv.")

    def __init__(self, micro_frame_size: Optional[int] = 17, micro_batch_size: Optional[int] = 4,
                 spatial_block_out_channels: Sequence[int] = (128, 256, 512, 512), scale=SCALE, shift=SHIFT):
        super().__init__()
        check_widths(spatial_block_out_channels, f"spatial_block_out_channels={tuple(spatial_block_out_channels)}")
        self.spatial_vae = _SpatialEncoderHolder(micro_batch_size, spatial_block_out_channels)
        self.temporal_vae = VAE_TemporalEncoder()
        self.micro_frame_size = micro_frame_size
        self.register_buffer("scale", torch.tensor(scale)[None, :, None, None, None], persistent=False)
        self.register_buffer("shift", torch.tensor(shift)[None, :, None, None, None], persistent=False)

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, **kwargs):
        """A LOCAL snapshot of hpcai-tech/OpenSora-VAE-v1.2: the ``model.safetensors`` the decoder reads."""
        from ...utils.checkpoint import load_local_checkpoint

        _, sd = load_local_checkpoint(path, subfolder or "")
        enc = cls(**kwargs)
        enc.load_state_dict(sd)
        return enc

    def _dropped(self, key: str) -> bool:
        return not key.startswith(self._KEPT_PREFIXES)

    def load_state_dict(self, state_dict, strict: bool = True):
        for k in ("scale", "shift"):
            if k in state_dict:
                getattr(self, k).copy_(state_dict[k].reshape(getattr(self, k).shape))
        return super().load_state_dict(state_dict, strict=strict)

    @property
    def dtype(self):
        return self.temporal_vae.encoder.norm1.weight.dtype

    @property
    def device(self):
        return self.temporal_vae.encoder.norm1.weight.device

    @torch.no_grad()
    def encode(self, x):
        """x [B, 3, T, H, W] in [-1, 1] -> z [B, 4, T', H // 8, W // 8] = (sample - shift) / scale.

        Noise is drawn as the reference draws it, so a seeded caller consumes the generators in the same order and
        shapes: per image micro-batch ``torch.randn([n, 4, h, w], device, dtype)`` on the parameters' device (diffusers
        0.30's DiagonalGaussianDistribution.sample -> randn_tensor with generator None, models/autoencoders/vae.py),
        then per 17-frame chunk ``torch.randn([B, 4, t, h, w])`` on the CPU, moved to the device (:36-39)."""
        kernels.require_cuda(x, f"{type(self).__name__}.encode")
        x = x.to(self.dtype)
        kernels.require_cuda(x, f"{type(self).__name__}.encode", half_only=True)
        self._pack_weights()
        dev, dt = x.device, x.dtype
        B, _, T, H, W = x.shape
        # 1. the image encoder, micro_batch_size frames at a time (:503-520): latent_dist.sample() * 0.18215
        frames = x.permute(0, 2, 3, 4, 1).reshape(B * T, 1, H, W, 3)
        N = B * T
        bs = N if self.spatial_vae.micro_batch_size is None else self.spatial_vae.micro_batch_size
        parts = []
        for i in range(0, N, bs):
            m = self.spatial_vae.module.moments(pad_latent(frames[i:i + bs]))
            n, _, h, w, _ = m.shape
            noise = torch.randn(n, 4, h, w, device=dev, dtype=dt).permute(0, 2, 3, 1)[:, None]
            parts.append(_sample(m, noise) * SD_SCALING)
        x_z = torch.cat(parts).reshape(B, T, *parts[0].shape[2:])  # [B, T, h, w, 4]
        # 2. the temporal encoder per micro_frame_size frames (:656-665), posterior.sample() with CPU noise
        step = T if self.micro_frame_size is None else self.micro_frame_size
        zs = []
        for i in range(0, T, step):
            m = self.temporal_vae.moments(x_z[:, i:i + step])
            Bm, t, h, w, _ = m.shape
            noise = torch.randn(Bm, 4, t, h, w).to(device=dev, dtype=dt).permute(0, 2, 3, 4, 1)
            zs.append(_sample(m, noise))
        z = torch.cat(zs, dim=1).permute(0, 4, 1, 2, 3)
        # 3. (z - shift) / scale (:670)
        return (z - self.shift.to(z.dtype)) / self.scale.to(z.dtype)


def load_vae_encoder(encoder, vae=None, micro_batch_size: int = 4):
    """The native encoder of an ``OpenSoraConfig.vae_encoder`` value: an instance as it is, a local snapshot directory
    (its root or its ``vae/`` folder) loaded with ``micro_batch_size`` image frames per spatial pass; None stands for
    ``vae`` when that is a local directory.  Anything else: None."""
    if encoder is None:
        encoder = vae
    if isinstance(encoder, OpenSoraVAEEncoder):
        return encoder
    if isinstance(encoder, (str, os.PathLike)) and os.path.isdir(encoder):
        encoder = str(encoder)
        sub = "vae" if os.path.isdir(os.path.join(encoder, "vae")) else None
        return OpenSoraVAEEncoder.from_pretrained(encoder, subfolder=sub, micro_batch_size=micro_batch_size)
    return None


def load_vae(vae, micro_batch_size: int = 4):
    """The native decoder of an ``OpenSoraConfig.vae`` value: an instance as it is, a local snapshot directory (its root
    or its ``vae/`` folder) loaded with ``micro_batch_size`` image frames per spatial pass, anything else (the default
    hub id) None."""
    if isinstance(vae, VideoAutoencoderPipeline):
        return vae
    if isinstance(vae, (str, os.PathLike)) and os.path.isdir(vae):
        vae = str(vae)
        sub = "vae" if os.path.isdir(os.path.join(vae, "vae")) else None
        return VideoAutoencoderPipeline.from_pretrained(vae, subfolder=sub, micro_batch_size=micro_batch_size)
    return None
