"""diffusers' ``AutoencoderKL``, decoder half (diffusers 0.30: models/autoencoders/autoencoder_kl.py, the ``Decoder`` of
vae.py, ``UNetMidBlock2D`` / ``UpDecoderBlock2D`` of unets/unet_2d_blocks.py, ``ResnetBlock2D``, ``Upsample2D`` and the
mid-block ``Attention`` with ``AttnProcessor2_0``) on the sm_90a kernels of csrc/vae_conv.cu, with diffusers' parameter
names.  The image VAE of OpenSora v1.2 (SDXL), of Latte without the temporal decoder (sd-vae-ft-ema) and of
Vchitect-2.0 (16 latent channels, no ``post_quant_conv``, a ``shift_factor``).

``AutoencoderKL`` is the decoder half only: its ``encode`` raises ``NotImplementedError``.  The encoder half's blocks
(``SpatialEncoder``: diffusers' ``Encoder``, ``DownEncoderBlock2D`` and ``Downsample2D`` on the strided vae_conv_down)
serve the OpenSora v1.2 encoder (autoencoder_kl_open_sora.OpenSoraVAEEncoder).  Images are channels-last ``[N, 1, H, W, C]``
between kernels (T = 1, so each image is its own GroupNorm sample and the 3x3 convolutions are kt = 1); the latent is
zero padded to 16 channels; ``post_quant_conv`` and the 1x1 shortcuts are GEMMs on the pixel rows; the mid-block
attention is one GEMM for q | k | v, the materialised per-image softmax, and ``to_out`` with the residual in the GEMM
epilogue.  Every nonlinearity is ``nn.SiLU`` (``vae_groupnorm_act(act=2)``).
"""
from typing import Optional, Sequence

import torch
import torch.nn as nn

from ... import kernels
from ._common import DecoderOnlyVAE, attention, check_widths, group_norm, pad_1x1, pad_latent, run_conv

_SILU = 2  # vae_groupnorm_act's F.silu mode


class DecoderOutput:
    """diffusers.models.autoencoders.vae.DecoderOutput: ``.sample``."""

    def __init__(self, sample):
        self.sample = sample


class ResnetBlock2D(nn.Module):
    """norm1 -> SiLU -> conv1 -> norm2 -> SiLU -> conv2, out = (x + h) / 1.0 with x through the 1x1 ``conv_shortcut``
    (bias) where the width changes.  GroupNorm eps 1e-6."""

    def __init__(self, in_channels, out_channels, groups=32, eps=1e-6):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        if in_channels != out_channels:
            self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1)

    def forward(self, x):
        h = run_conv(self.conv1, group_norm(self.norm1, x, act=_SILU))
        n = group_norm(self.norm2, h, act=_SILU)
        if self.in_channels != self.out_channels:
            x = kernels.gemm_bias_act(x, self.conv_shortcut._w, self.conv_shortcut._b)
        return run_conv(self.conv2, n, resid=x)  # dividing by output_scale_factor = 1.0 is exact


class Attention(nn.Module):
    """The mid block's single-head attention (heads = 1, dim_head = C): group_norm, to_q / to_k / to_v, softmax(Q K^T *
    C^-0.5) V over each frame's pixels, to_out.0, + residual."""

    def __init__(self, channels, groups=32, eps=1e-6):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, channels, eps=eps, affine=True)
        self.to_q = nn.Linear(channels, channels)
        self.to_k = nn.Linear(channels, channels)
        self.to_v = nn.Linear(channels, channels)
        self.to_out = nn.ModuleList([nn.Linear(channels, channels), nn.Dropout(0.0)])
        self._w_qkv = self._b_qkv = None

    def pack(self):
        self._w_qkv = torch.cat([self.to_q.weight, self.to_k.weight, self.to_v.weight]).detach().contiguous()
        self._b_qkv = torch.cat([self.to_q.bias, self.to_k.bias, self.to_v.bias]).detach().contiguous()

    def forward(self, x):
        out = self.to_out[0]
        return attention(x, self.group_norm, self._w_qkv, self._b_qkv, out.weight, out.bias, False)


class UNetMidBlock2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(channels, channels), ResnetBlock2D(channels, channels)])
        self.attentions = nn.ModuleList([Attention(channels)])

    def forward(self, x):
        return self.resnets[1](self.attentions[0](self.resnets[0](x)))


class Upsample2D(nn.Module):
    """Nearest 2x in H and W, then a 3x3 ``conv`` (the fp32 up-cast around the interpolation is exact)."""

    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)

    def forward(self, x):
        return run_conv(self.conv, kernels.vae_upsample2x(x, False))


class UpDecoderBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(in_channels if i == 0 else out_channels, out_channels)
                                      for i in range(num_layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(out_channels)]) if add_upsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class SpatialDecoder(nn.Module):
    """diffusers' ``Decoder``: conv_in, mid_block, up_blocks (widest first, layers_per_block + 1 resnets each, nearest
    up-sampling after all but the last), conv_norm_out (eps 1e-6) + SiLU, conv_out."""

    def __init__(self, latent_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2):
        super().__init__()
        rev = list(reversed(block_out_channels))
        self.conv_in = nn.Conv2d(latent_channels, rev[0], 3, padding=1)
        self.mid_block = UNetMidBlock2D(rev[0])
        self.up_blocks = nn.ModuleList([])
        prev = rev[0]
        for i, ch in enumerate(rev):
            self.up_blocks.append(UpDecoderBlock2D(prev, ch, layers_per_block + 1, add_upsample=i < len(rev) - 1))
            prev = ch
        self.conv_norm_out = nn.GroupNorm(32, block_out_channels[0], eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], out_channels, 3, padding=1)

    def forward(self, z):
        """z [N, 1, h, w, 16] (frames in the batch, zero padded) -> [N, 1, 8h, 8w, 3]."""
        x = self.mid_block(run_conv(self.conv_in, z))
        for up in self.up_blocks:
            x = up(x)
        return run_conv(self.conv_out, group_norm(self.conv_norm_out, x, act=_SILU))


class Downsample2D(nn.Module):
    """diffusers' Downsample2D with use_conv and padding 0: F.pad(x, (0, 1, 0, 1)), then a 3x3 ``conv`` with stride 2
    (vae_conv_down, the padding being its out-of-bounds fill)."""

    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=0)

    def forward(self, x):
        return kernels.vae_conv_down(x, self.conv._w, self.conv._b, self.conv.out_channels, 1)


class DownEncoderBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(in_channels if i == 0 else out_channels, out_channels)
                                      for i in range(num_layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(out_channels)]) if add_downsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
        return x


class SpatialEncoder(nn.Module):
    """diffusers' ``Encoder`` (double_z): conv_in, down_blocks (layers_per_block resnets each, a stride-2 down-sampling
    after all but the last), mid_block, conv_norm_out (eps 1e-6) + SiLU, conv_out to 2 * latent_channels."""

    def __init__(self, in_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512), layers_per_block=2):
        super().__init__()
        self.conv_in = nn.Conv2d(in_channels, block_out_channels[0], 3, padding=1)
        self.down_blocks = nn.ModuleList([])
        prev = block_out_channels[0]
        for i, ch in enumerate(block_out_channels):
            self.down_blocks.append(DownEncoderBlock2D(prev, ch, layers_per_block, add_downsample=i < len(block_out_channels) - 1))
            prev = ch
        self.mid_block = UNetMidBlock2D(prev)
        self.conv_norm_out = nn.GroupNorm(32, prev, eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(prev, 2 * latent_channels, 3, padding=1)

    def forward(self, x):
        """x [N, 1, H, W, 16] (images in the batch, RGB zero padded) -> moments [N, 1, h, w, 2 * latent_channels]."""
        x = run_conv(self.conv_in, x)
        for down in self.down_blocks:
            x = down(x)
        return run_conv(self.conv_out, group_norm(self.conv_norm_out, self.mid_block(x), act=_SILU))


class AutoencoderKL(DecoderOnlyVAE):
    """diffusers' AutoencoderKL, decoder half (``post_quant_conv`` when ``use_post_quant_conv``, ``decoder``).  The SDXL
    and sd-vae-ft-ema VAEs have block_out_channels (128, 256, 512, 512), layers_per_block 2, latent_channels 4;
    Vchitect-2.0's has latent_channels 16 and no post_quant_conv.  ``load_state_dict`` drops ``encoder.*`` and
    ``quant_conv.*`` and is strict about every other key."""

    _DROPPED_PREFIXES = ("encoder.", "quant_conv.")

    def __init__(self, in_channels: int = 3, out_channels: int = 3,
                 up_block_types: Optional[Sequence[str]] = None,
                 block_out_channels: Sequence[int] = (128, 256, 512, 512), layers_per_block: int = 2, act_fn: str = "silu",
                 latent_channels: int = 4, norm_num_groups: int = 32, sample_size: int = 32,
                 scaling_factor: float = 0.18215, shift_factor: Optional[float] = None, force_upcast: bool = True,
                 use_quant_conv: bool = True, use_post_quant_conv: bool = True, mid_block_add_attention: bool = True):
        super().__init__()
        up_block_types = tuple(up_block_types) if up_block_types is not None else ("UpDecoderBlock2D",) * len(block_out_channels)
        if any(t != "UpDecoderBlock2D" for t in up_block_types) or len(up_block_types) != len(block_out_channels):
            raise NotImplementedError(f"up_block_types={up_block_types}: only UpDecoderBlock2D, one per width, is built")
        if not mid_block_add_attention:
            raise NotImplementedError("mid_block_add_attention=False is not built (the released VAEs have the attention)")
        if norm_num_groups != 32:
            raise NotImplementedError(f"norm_num_groups={norm_num_groups}: the decoder is built with 32 groups")
        if act_fn not in ("silu", "swish"):
            raise NotImplementedError(f"act_fn={act_fn!r}: the decoder kernels apply SiLU")
        if out_channels != 3:
            raise NotImplementedError(f"out_channels={out_channels}: the decoder writes RGB")
        if not 1 <= latent_channels <= 16:
            raise NotImplementedError(f"latent_channels={latent_channels}: the latent is padded to 16 channels")
        check_widths(block_out_channels, f"block_out_channels={tuple(block_out_channels)}")
        self.config = type("Config", (), dict(
            in_channels=in_channels, out_channels=out_channels, up_block_types=up_block_types,
            block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block, act_fn=act_fn,
            latent_channels=latent_channels, norm_num_groups=norm_num_groups, sample_size=sample_size,
            scaling_factor=scaling_factor, shift_factor=shift_factor, force_upcast=force_upcast,
            use_quant_conv=use_quant_conv, use_post_quant_conv=use_post_quant_conv,
            mid_block_add_attention=mid_block_add_attention))()
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1) if use_post_quant_conv else None
        self.decoder = SpatialDecoder(latent_channels, 3, block_out_channels, layers_per_block)
        self._pq = None

    @classmethod
    def from_pretrained(cls, path: str, subfolder: str = "vae"):
        """A LOCAL diffusers snapshot (``<path>/<subfolder>/config.json`` + weights); no hub download."""
        return cls._from_local_diffusers(path, subfolder)

    @property
    def dtype(self):
        return self.decoder.conv_in.weight.dtype

    @property
    def device(self):
        return self.decoder.conv_in.weight.device

    def pack(self):
        if self.post_quant_conv is not None:
            self._pq = pad_1x1(self.post_quant_conv.weight, self.post_quant_conv.bias)

    def decode_frames(self, z):
        """z [N, 1, h, w, 16] (channels-last, zero padded) -> [N, 1, 8h, 8w, 3]."""
        return self.decoder(kernels.gemm_bias_act(z, *self._pq) if self.post_quant_conv is not None else z)

    @torch.no_grad()
    def decode(self, z, return_dict: bool = True):
        """z [N, latent_channels, h, w] (already scaled as the caller's pipeline does) -> ``.sample`` [N, 3, 8h, 8w]."""
        z = self._decode_input(z)
        x = self.decode_frames(pad_latent(z.permute(0, 2, 3, 1))[:, None])
        dec = x[:, 0].permute(0, 3, 1, 2)
        return DecoderOutput(sample=dec) if return_dict else (dec,)
