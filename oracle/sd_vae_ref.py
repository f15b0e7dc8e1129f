"""TEST INFRASTRUCTURE ONLY -- a CPU restatement of the decode path of diffusers' ``AutoencoderKL`` (the SDXL image VAE
that OpenSora v1.2's ``VideoAutoencoderKL`` loads from ``PixArt-alpha/pixart_sigma_sdxlvae_T5_diffusers``).

diffusers is not installed here, so the module cannot be imported; this file restates, in plain eager torch, the facts of
diffusers' ``AutoencoderKL`` / ``Decoder`` / ``UNetMidBlock2D`` / ``UpDecoderBlock2D`` / ``ResnetBlock2D`` /
``Upsample2D`` / ``Attention`` (``AttnProcessor2_0``) that the decode path uses, with diffusers' parameter names:
  - ``post_quant_conv``: 1x1 Conv2d latent -> latent channels;
  - ``decoder.conv_in``: 3x3 Conv2d latent -> block_out_channels[-1];
  - ``decoder.mid_block``: ``resnets.0``, ``attentions.0``, ``resnets.1``;
  - ``decoder.up_blocks.{i}`` over reversed(block_out_channels): layers_per_block + 1 ``resnets`` each, the first taking
    the previous block's width; all but the last end in ``upsamplers.0``: nearest 2x, then a 3x3 ``conv``;
  - ``decoder.conv_norm_out`` GroupNorm(32, block_out_channels[0], eps 1e-6), ``conv_act`` SiLU, ``conv_out`` 3x3 -> 3;
  - ``ResnetBlock2D``: norm1 -> SiLU -> conv1 -> norm2 -> SiLU -> conv2, ``conv_shortcut`` (1x1, bias) where the width
    changes, out = (shortcut + h) / 1.0; GroupNorm(32, eps 1e-6);
  - mid-block ``Attention``: one head of dim block_out_channels[-1]; ``group_norm`` (32, eps 1e-6) over each image's
    pixels, ``to_q`` / ``to_k`` / ``to_v`` Linear with bias, scaled_dot_product_attention (scale dim^-0.5),
    ``to_out.0`` Linear with bias, + residual, / 1.0.
Only the decoder exists here (``encode`` is out of scope, as in the product)."""
import types

import torch
import torch.nn as nn
import torch.nn.functional as F


class ResnetBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, in_channels, eps=1e-6)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.norm2 = nn.GroupNorm(32, out_channels, eps=1e-6)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None

    def forward(self, x):
        h = self.conv1(F.silu(self.norm1(x)))
        h = self.conv2(F.silu(self.norm2(h)))
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return (x + h) / 1.0


class Attention(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.group_norm = nn.GroupNorm(32, channels, eps=1e-6)
        self.to_q = nn.Linear(channels, channels)
        self.to_k = nn.Linear(channels, channels)
        self.to_v = nn.Linear(channels, channels)
        self.to_out = nn.ModuleList([nn.Linear(channels, channels), nn.Dropout(0.0)])

    def forward(self, x):
        residual = x
        B, C, H, W = x.shape
        h = self.group_norm(x.view(B, C, H * W)).transpose(1, 2)
        q, k, v = (m(h)[:, None] for m in (self.to_q, self.to_k, self.to_v))  # [B, heads = 1, HW, C]
        o = F.scaled_dot_product_attention(q, k, v)[:, 0].to(q.dtype)
        o = self.to_out[1](self.to_out[0](o))
        return (o.transpose(1, 2).reshape(B, C, H, W) + residual) / 1.0


class UNetMidBlock2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(channels, channels), ResnetBlock2D(channels, channels)])
        self.attentions = nn.ModuleList([Attention(channels)])

    def forward(self, x):
        return self.resnets[1](self.attentions[0](self.resnets[0](x)))


class Upsample2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)

    def forward(self, x):
        dtype = x.dtype
        x = F.interpolate(x.float(), scale_factor=2.0, mode="nearest").to(dtype)
        return self.conv(x)


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


class Decoder(nn.Module):
    def __init__(self, latent_channels, block_out_channels, layers_per_block):
        super().__init__()
        rev = list(reversed(block_out_channels))
        self.conv_in = nn.Conv2d(latent_channels, rev[0], 3, padding=1)
        self.mid_block = UNetMidBlock2D(rev[0])
        self.up_blocks = nn.ModuleList()
        prev = rev[0]
        for i, ch in enumerate(rev):
            self.up_blocks.append(UpDecoderBlock2D(prev, ch, layers_per_block + 1, i < len(rev) - 1))
            prev = ch
        self.conv_norm_out = nn.GroupNorm(32, block_out_channels[0], eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], 3, 3, padding=1)

    def forward(self, z):
        x = self.mid_block(self.conv_in(z))
        for up in self.up_blocks:
            x = up(x)
        return self.conv_out(self.conv_act(self.conv_norm_out(x)))


class AutoencoderKL(nn.Module):
    """decoder half of diffusers' AutoencoderKL; ``decode(z).sample`` as diffusers returns it."""

    def __init__(self, block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4):
        super().__init__()
        self.config = types.SimpleNamespace(block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                            latent_channels=latent_channels)
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)
        self.decoder = Decoder(latent_channels, block_out_channels, layers_per_block)

    def decode(self, z):
        return types.SimpleNamespace(sample=self.decoder(self.post_quant_conv(z)))
