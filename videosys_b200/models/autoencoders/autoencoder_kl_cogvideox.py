"""CogVideoX VAE decoder (mirror of videosys/models/autoencoders/autoencoder_kl_cogvideox.py: AutoencoderKLCogVideoX
:872-1239 and the decoder modules it builds, :59-299, :408-594, :731-869; CogVideoXUpsample3D, models/modules/
upsampling.py:6-67) on the sm_90a kernels of csrc/vae_conv.cu.

Only the decoder is in scope: ``encode`` raises ``NotImplementedError``.  The module keeps the reference's parameter names
and shapes under ``decoder.*``.  Activations stay channels-last ``[B, T, H, W, C]`` between kernels:
  - every causal convolution (``conv_in``, ``conv1`` / ``conv2`` of each ResNet, ``conv_out``) reads a buffer that holds
    its two causal context frames first (copies of frame 0 for the first frame batch, else the conv cache carried from
    the previous batch, reference :112-129), then the frames the spatial norm + SiLU kernel wrote;
  - the spatial norm's ``conv_y`` / ``conv_b`` (1x1x1, 16 -> C) run as one GEMM at latent resolution; the kernel gathers
    their result with the nearest-interpolation rule (equal to interpolating first, because the conv is per pixel);
  - ``conv_shortcut`` (1x1x1) is a GEMM on the pixel rows; the ResNet sum is the conv2 epilogue.
The frame batching of ``_decode`` and the tiling of ``tiled_decode`` reproduce the reference's integer arithmetic.
"""
from typing import Optional, Tuple

import torch
import torch.nn as nn

from ... import kernels
from ._common import DecoderOnlyVAE, check_widths, conv_buffer, run_conv, tiled_decode_2d


class DecoderOutput:
    """diffusers.models.autoencoders.vae.DecoderOutput: ``.sample``."""

    def __init__(self, sample):
        self.sample = sample


class CogVideoXCausalConv3d(nn.Module):
    """Reference :59-135 with kernel (kt, 3, 3), stride 1 (kt = 1 for the spatial norm's conv_y / conv_b)."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size: int):
        super().__init__()
        self.time_kernel_size = kernel_size
        self.conv = nn.Conv3d(in_channels, out_channels, kernel_size)
        self.conv_cache = None

    def _clear_fake_context_parallel_cache(self):
        self.conv_cache = None

    def input_buffer(self, x_shape, dtype, device):
        return conv_buffer(self.conv, x_shape, dtype, device)

    def run(self, buf, resid=None):
        """Fills the two context frames of buf, keeps the new cache, and convolves (reference :123-135)."""
        if self.conv_cache is None:
            buf[:, :2] = buf[:, 2:3]
        else:
            buf[:, :2] = self.conv_cache
        self.conv_cache = buf[:, -2:].clone()
        return run_conv(self.conv, buf, resid)


class CogVideoXSpatialNorm3D(nn.Module):
    """Reference :138-178, followed by SiLU."""

    def __init__(self, f_channels: int, zq_channels: int, groups: int = 32):
        super().__init__()
        self.norm_layer = nn.GroupNorm(num_channels=f_channels, num_groups=groups, eps=1e-6, affine=True)
        self.conv_y = CogVideoXCausalConv3d(zq_channels, f_channels, kernel_size=1)
        self.conv_b = CogVideoXCausalConv3d(zq_channels, f_channels, kernel_size=1)
        self._w = self._b = None

    def pack(self):
        self._w = torch.cat([self.conv_y.conv.weight, self.conv_b.conv.weight]).flatten(1).detach().contiguous()
        self._b = torch.cat([self.conv_y.conv.bias, self.conv_b.conv.bias]).detach().contiguous()

    def norm_silu_into(self, f, zq, buf):
        """silu(norm(f, zq)) of f [B, T, H, W, C] into frames 2.. of buf; zq [B, Tz, h, w, Cz] is the latent frame batch."""
        zyb = kernels.gemm_bias_act(zq, self._w, self._b)  # [B, Tz, h, w, 2C] = conv_y | conv_b
        stats = kernels.vae_groupnorm_stats(f, self.norm_layer.num_groups, self.norm_layer.eps)
        return kernels.vae_spatial_norm_silu(f, stats, self.norm_layer.weight, self.norm_layer.bias, zyb, buf, t_off=2)


class CogVideoXResnetBlock3D(nn.Module):
    """Reference :181-299 with spatial norms, no time embedding, dropout 0."""

    def __init__(self, in_channels: int, out_channels: int, groups: int, zq_channels: int):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = CogVideoXSpatialNorm3D(in_channels, zq_channels, groups)
        self.norm2 = CogVideoXSpatialNorm3D(out_channels, zq_channels, groups)
        self.conv1 = CogVideoXCausalConv3d(in_channels, out_channels, 3)
        self.conv2 = CogVideoXCausalConv3d(out_channels, out_channels, 3)
        if in_channels != out_channels:
            self.conv_shortcut = nn.Conv3d(in_channels, out_channels, kernel_size=1)

    def forward(self, x, zq):
        buf = self.conv1.input_buffer(x.shape, x.dtype, x.device)
        h = self.conv1.run(self.norm1.norm_silu_into(x, zq, buf))
        buf = self.conv2.input_buffer(h.shape, h.dtype, h.device)
        self.norm2.norm_silu_into(h, zq, buf)
        if self.in_channels != self.out_channels:
            x = kernels.gemm_bias_act(x, self.conv_shortcut._w, self.conv_shortcut._b)
        return self.conv2.run(buf, resid=x)


class CogVideoXUpsample3D(nn.Module):
    """modules/upsampling.py:6-67: nearest 2x (and in time with compress_time), then a 3x3 Conv2d per frame."""

    def __init__(self, in_channels: int, out_channels: int, compress_time: bool = False):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.compress_time = compress_time

    def forward(self, x):
        return run_conv(self.conv, kernels.vae_upsample2x(x, self.compress_time))


class CogVideoXMidBlock3D(nn.Module):
    def __init__(self, channels: int, groups: int, zq_channels: int, num_layers: int = 2):
        super().__init__()
        self.resnets = nn.ModuleList([CogVideoXResnetBlock3D(channels, channels, groups, zq_channels) for _ in range(num_layers)])

    def forward(self, x, zq):
        for r in self.resnets:
            x = r(x, zq)
        return x


class CogVideoXUpBlock3D(nn.Module):
    def __init__(self, in_channels: int, out_channels: int, groups: int, zq_channels: int, num_layers: int, add_upsample: bool,
                 compress_time: bool):
        super().__init__()
        self.resnets = nn.ModuleList([CogVideoXResnetBlock3D(in_channels if i == 0 else out_channels, out_channels, groups, zq_channels)
                                      for i in range(num_layers)])
        self.upsamplers = nn.ModuleList([CogVideoXUpsample3D(out_channels, out_channels, compress_time)]) if add_upsample else None

    def forward(self, x, zq):
        for r in self.resnets:
            x = r(x, zq)
        if self.upsamplers is not None:
            for u in self.upsamplers:
                x = u(x)
        return x


class CogVideoXDecoder3D(nn.Module):
    """Reference :731-869."""

    def __init__(self, in_channels: int = 16, out_channels: int = 3, block_out_channels: Tuple[int, ...] = (128, 256, 256, 512),
                 layers_per_block: int = 3, norm_num_groups: int = 32, temporal_compression_ratio: float = 4):
        super().__init__()
        import math

        rev = list(reversed(block_out_channels))
        self.conv_in = CogVideoXCausalConv3d(in_channels, rev[0], 3)
        self.mid_block = CogVideoXMidBlock3D(rev[0], norm_num_groups, in_channels)
        self.up_blocks = nn.ModuleList([])
        level = int(math.log2(temporal_compression_ratio))
        out_c = rev[0]
        for i in range(len(block_out_channels)):
            prev, out_c = out_c, rev[i]
            self.up_blocks.append(CogVideoXUpBlock3D(prev, out_c, norm_num_groups, in_channels, layers_per_block + 1,
                                                     add_upsample=i != len(block_out_channels) - 1, compress_time=i < level))
        self.norm_out = CogVideoXSpatialNorm3D(rev[-1], in_channels, norm_num_groups)
        self.conv_out = CogVideoXCausalConv3d(rev[-1], out_channels, 3)

    def forward(self, sample):
        """sample [B, Cz, T, h, w] -> [B, out_channels, T', 8h, 8w] (one frame batch; conv caches carried)."""
        zq = sample.permute(0, 2, 3, 4, 1).contiguous()  # [B, T, h, w, Cz]
        buf = self.conv_in.input_buffer(zq.shape, zq.dtype, zq.device)
        buf[:, 2:] = zq
        x = self.conv_in.run(buf)
        x = self.mid_block(x, zq)
        for ub in self.up_blocks:
            x = ub(x, zq)
        buf = self.conv_out.input_buffer(x.shape, x.dtype, x.device)
        self.norm_out.norm_silu_into(x, zq, buf)
        return self.conv_out.run(buf).permute(0, 4, 1, 2, 3)


class AutoencoderKLCogVideoX(DecoderOnlyVAE):
    """Reference :872-1239, decoder only.  ``load_state_dict`` drops the ``encoder.*`` and ``quant_conv.*`` entries of the
    reference's full state dict."""

    _DROPPED_PREFIXES = ("encoder.", "quant_conv.")

    def __init__(self, in_channels: int = 3, out_channels: int = 3,
                 down_block_types: Tuple[str] = ("CogVideoXDownBlock3D",) * 4,
                 up_block_types: Tuple[str] = ("CogVideoXUpBlock3D",) * 4,
                 block_out_channels: Tuple[int] = (128, 256, 256, 512), latent_channels: int = 16, layers_per_block: int = 3,
                 act_fn: str = "silu", norm_eps: float = 1e-6, norm_num_groups: int = 32, temporal_compression_ratio: float = 4,
                 sample_height: int = 480, sample_width: int = 720, scaling_factor: float = 1.15258426,
                 shift_factor: Optional[float] = None, latents_mean: Optional[Tuple[float]] = None,
                 latents_std: Optional[Tuple[float]] = None, force_upcast: float = True, use_quant_conv: bool = False,
                 use_post_quant_conv: bool = False):
        super().__init__()
        if use_post_quant_conv:
            raise NotImplementedError("use_post_quant_conv=True is not supported (the released CogVideoX VAE has none)")
        if any(t != "CogVideoXUpBlock3D" for t in up_block_types):
            raise ValueError("Invalid `up_block_type` encountered. Must be `CogVideoXUpBlock3D`")
        if len(up_block_types) != len(block_out_channels):
            raise ValueError("up_block_types and block_out_channels must have the same length")
        if act_fn not in ("silu", "swish"):
            raise ValueError(f"act_fn={act_fn!r}: the decoder kernels apply SiLU")
        check_widths(block_out_channels, f"block_out_channels {tuple(block_out_channels)}")
        for c in block_out_channels:
            if c % norm_num_groups:
                raise ValueError(f"norm_num_groups={norm_num_groups} does not divide {c} channels")
        if not (latent_channels == 16 or latent_channels % 64 == 0):
            raise ValueError(f"latent_channels={latent_channels}: the convolution takes 16 or a multiple of 64")
        if not (out_channels == 3 or out_channels % 64 == 0):
            raise ValueError(f"out_channels={out_channels}: the convolution takes 3 or a multiple of 64")
        self.config = type("Config", (), dict(
            in_channels=in_channels, out_channels=out_channels, down_block_types=tuple(down_block_types),
            up_block_types=tuple(up_block_types), block_out_channels=tuple(block_out_channels), latent_channels=latent_channels,
            layers_per_block=layers_per_block, act_fn=act_fn, norm_eps=norm_eps, norm_num_groups=norm_num_groups,
            temporal_compression_ratio=temporal_compression_ratio, sample_height=sample_height, sample_width=sample_width,
            scaling_factor=scaling_factor, shift_factor=shift_factor, latents_mean=latents_mean, latents_std=latents_std,
            force_upcast=force_upcast, use_quant_conv=use_quant_conv, use_post_quant_conv=use_post_quant_conv))()
        self.decoder = CogVideoXDecoder3D(latent_channels, out_channels, tuple(block_out_channels), layers_per_block,
                                          norm_num_groups, temporal_compression_ratio)
        self.post_quant_conv = None
        self.use_slicing = False
        self.use_tiling = False
        self.num_latent_frames_batch_size = 2
        self.tile_sample_min_height = sample_height // 2
        self.tile_sample_min_width = sample_width // 2
        self.tile_latent_min_height = int(self.tile_sample_min_height / (2 ** (len(block_out_channels) - 1)))
        self.tile_latent_min_width = int(self.tile_sample_min_width / (2 ** (len(block_out_channels) - 1)))
        self.tile_overlap_factor_height = 1 / 6
        self.tile_overlap_factor_width = 1 / 5

    @classmethod
    def from_pretrained(cls, path: str, subfolder: str = "vae"):
        """A LOCAL snapshot directory (``<path>/<subfolder>/config.json`` + weights); no hub download."""
        return cls._from_local_diffusers(path, subfolder)

    @property
    def dtype(self):
        return self.decoder.conv_in.conv.weight.dtype

    # ---- reference switches (:1007-1068) ----
    def _clear_fake_context_parallel_cache(self):
        for m in self.modules():
            if isinstance(m, CogVideoXCausalConv3d):
                m._clear_fake_context_parallel_cache()

    def enable_tiling(self, tile_sample_min_height: Optional[int] = None, tile_sample_min_width: Optional[int] = None,
                      tile_overlap_factor_height: Optional[float] = None, tile_overlap_factor_width: Optional[float] = None):
        self.use_tiling = True
        self.tile_sample_min_height = tile_sample_min_height or self.tile_sample_min_height
        self.tile_sample_min_width = tile_sample_min_width or self.tile_sample_min_width
        n = 2 ** (len(self.config.block_out_channels) - 1)
        self.tile_latent_min_height = int(self.tile_sample_min_height / n)
        self.tile_latent_min_width = int(self.tile_sample_min_width / n)
        self.tile_overlap_factor_height = tile_overlap_factor_height or self.tile_overlap_factor_height
        self.tile_overlap_factor_width = tile_overlap_factor_width or self.tile_overlap_factor_width

    def disable_tiling(self):
        self.use_tiling = False

    def enable_slicing(self):
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False

    # ---- decoding (:1094-1239) ----
    def _decode_frame_batches(self, z):
        """The decoder over z's frame batches (the first one takes the remainder), the conv caches carried from batch to
        batch and cleared after the last."""
        fbs = self.num_latent_frames_batch_size
        num_frames = z.shape[2]
        rem = num_frames % fbs
        dec = [self.decoder(z[:, :, fbs * i + (0 if i == 0 else rem):fbs * (i + 1) + rem]) for i in range(num_frames // fbs)]
        self._clear_fake_context_parallel_cache()
        return torch.cat(dec, dim=2)

    def _decode(self, z, return_dict: bool = True):
        batch_size, num_channels, num_frames, height, width = z.shape
        if self.use_tiling and (width > self.tile_latent_min_width or height > self.tile_latent_min_height):
            return self.tiled_decode(z, return_dict=return_dict)
        dec = self._decode_frame_batches(z)
        return DecoderOutput(sample=dec) if return_dict else (dec,)

    @torch.no_grad()
    def decode(self, z, return_dict: bool = True):
        """z [B, latent_channels, T, h, w] (already divided by scaling_factor) -> [B, out_channels, 4 (T - 1) + 1, 8h, 8w]."""
        z = self._decode_input(z)
        if self.use_slicing and z.shape[0] > 1:
            decoded = torch.cat([self._decode(s).sample for s in z.split(1)])
        else:
            decoded = self._decode(z).sample
        return DecoderOutput(sample=decoded) if return_dict else (decoded,)

    def tiled_decode(self, z, return_dict: bool = True):
        dec = tiled_decode_2d(z, self._decode_frame_batches, (self.tile_latent_min_height, self.tile_latent_min_width),
                              (self.tile_sample_min_height, self.tile_sample_min_width),
                              (self.tile_overlap_factor_height, self.tile_overlap_factor_width))
        return DecoderOutput(sample=dec) if return_dict else (dec,)
