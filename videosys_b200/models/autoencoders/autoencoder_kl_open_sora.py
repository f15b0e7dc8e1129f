"""OpenSora v1.2 VAE decoder (mirror of videosys/models/autoencoders/autoencoder_kl_open_sora.py: CausalConv3d :89-124,
ResBlock :127-164, Decoder :275-376, VAE_Temporal :379-471, VAE_Temporal_SD :474-485, VideoAutoencoderKL :488-555,
VideoAutoencoderPipeline :621-729) on the sm_90a kernels of csrc/vae_conv.cu and csrc/vae_osp.cu.

Only the decoder is in scope: ``encode`` raises ``NotImplementedError``.  ``decode(z, num_frames)`` runs the reference's
three stages:
  1. ``z * scale + shift`` (persistent buffers, so a checkpoint's values load over the released ones);
  2. the temporal decoder (``temporal_vae``) per micro-batch of ``micro_z_frame_size`` = 5 latent frames, each chunk on its
     own (no causal state between chunks), with its leading ``time_padding`` frames trimmed;
  3. the SDXL image decoder (``spatial_vae.module``, diffusers' ``AutoencoderKL`` restated: diffusers' parameter names)
     on ``micro_batch_size`` frames at a time, each frame its own GroupNorm sample, after ``x / 0.18215``.
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
from .autoencoder_kl_open_sora_plan import _GN_CHANNELS, _LATENT_PAD

_SILU = 2  # vae_groupnorm_act's F.silu mode
SCALE = (3.85, 2.32, 2.33, 3.06)  # OpenSoraVAE_V1_2 (:748-749)
SHIFT = (-0.10, 0.34, 0.27, 0.98)
SD_SCALING = 0.18215  # VideoAutoencoderKL.decode divides the latent by this (:534)


def _cast_tuple(t, length=1):
    return tuple(t) if isinstance(t, (tuple, list)) else (t,) * length


def _gn(norm, x, out=None, t_off=0, act=_SILU):
    stats = kernels.vae_groupnorm_stats(x, norm.num_groups, norm.eps)
    return kernels.vae_groupnorm_act(x, stats, norm.weight, norm.bias, out=out, t_off=t_off, act=act)


def _pad_latent(z):
    """[..., c] (c <= 16) -> [..., 16], zero channels after c: the smallest Cin the convolution and the GEMM take."""
    zp = torch.zeros(*z.shape[:-1], _LATENT_PAD, dtype=z.dtype, device=z.device)
    zp[..., :z.shape[-1]] = z
    return zp


def _pad_1x1(weight, bias):
    """A 4 -> 4 1x1 convolution as a [16, 16] GEMM weight and a [16] bias (zero rows / columns)."""
    cout, cin = weight.shape[:2]
    w = torch.zeros(_LATENT_PAD, _LATENT_PAD, dtype=weight.dtype, device=weight.device)
    w[:cout, :cin] = weight.detach().flatten(1)
    b = torch.zeros(_LATENT_PAD, dtype=weight.dtype, device=weight.device)
    b[:cout] = bias.detach()
    return w, b


def _dropped(key: str) -> bool:
    """Encoder-side keys of the full checkpoint (``*.encoder.*``, ``*.quant_conv.*``): not part of the decoder."""
    parts = key.split(".")
    return "encoder" in parts or "quant_conv" in parts


# =====================================================================================================================
# temporal decoder (VAE_Temporal_SD)
# =====================================================================================================================
class CausalConv3d(nn.Module):
    """Reference :89-124: kt - 1 leading ZERO frames, zero spatial padding, then nn.Conv3d (``conv.*``)."""

    def __init__(self, chan_in, chan_out, kernel_size, bias=True):
        super().__init__()
        kernel_size = _cast_tuple(kernel_size, 3)
        self.chan_in, self.chan_out = chan_in, chan_out
        self.time_kernel_size = kernel_size[0]
        self.conv = nn.Conv3d(chan_in, chan_out, kernel_size, bias=bias)
        self._w = self._b = None

    def pack(self):
        w = self.conv.weight.detach()
        self._w = kernels.pack_conv_weight(w) if w.shape[-1] == 3 else w.flatten(1).contiguous()
        b = self.conv.bias
        self._b = b.detach() if b is not None else torch.zeros(self.chan_out, dtype=w.dtype, device=w.device)

    def input_buffer(self, x_shape, dtype, device):
        """[B, kt - 1 + T, H, W, Cin] with the kt - 1 context frames zeroed: frames kt - 1 .. are the caller's."""
        B, T, H, W, C = x_shape
        ctx = self.time_kernel_size - 1
        buf = torch.empty(B, ctx + T, H, W, C, dtype=dtype, device=device)
        buf[:, :ctx].zero_()
        return buf

    def run(self, buf, resid=None):
        # bias-free convolutions carry a zero bias: bf16(conv + 0) is the rounded convolution
        return kernels.vae_conv3d(buf, self._w, self._b, self.chan_out, self.time_kernel_size, resid=resid, round_conv=True)


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
        _gn(self.norm1, x, buf, t_off=2)
        h = self.conv1.run(buf)
        buf = self.conv2.input_buffer(h.shape, h.dtype, h.device)
        _gn(self.norm2, h, buf, t_off=2)
        if self.in_channels != self.filters:
            x = kernels.gemm_bias_act(x, self.conv3._w)
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
        _gn(self.norm1, x, buf, t_off=2)
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


# =====================================================================================================================
# image decoder: diffusers AutoencoderKL (Decoder, UNetMidBlock2D, UpDecoderBlock2D, ResnetBlock2D, Upsample2D,
# Attention with AttnProcessor2_0), decoder half, with diffusers' parameter names
# =====================================================================================================================
def _conv2d_pack(conv):
    conv._w = kernels.pack_conv_weight(conv.weight.detach())
    conv._b = conv.bias.detach()


def _conv2d_run(conv, x, resid=None):
    """A 3x3 Conv2d (padding 1, bias) of x [N, 1, H, W, Cin] -> [N, 1, H, W, Cout]."""
    return kernels.vae_conv3d(x, conv._w, conv._b, conv.out_channels, 1, resid=resid, round_conv=True)


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
        h = _conv2d_run(self.conv1, _gn(self.norm1, x))
        n = _gn(self.norm2, h)
        if self.in_channels != self.out_channels:
            x = kernels.gemm_bias_act(x, self.conv_shortcut._w, self.conv_shortcut.bias)
        return _conv2d_run(self.conv2, n, resid=x)  # dividing by output_scale_factor = 1.0 is exact


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

    def forward(self, x):
        N, T, H, W, C = x.shape
        qkv = kernels.gemm_bias_act(_gn(self.group_norm, x, act=False), self._w_qkv, self._b_qkv)
        q, k, vt = kernels.vae_attn_split(qkv, C, False)
        P, Pp = H * W, k.shape[1]
        o = torch.empty(N * T, P, C, dtype=x.dtype, device=x.device)
        s = torch.empty(P, Pp, dtype=x.dtype, device=x.device)  # one frame's scores at a time
        for f in range(N * T):
            kernels.gemm_bias_act(q[f], k[f], out=s)
            kernels.vae_attn_softmax_(s, P, int(C) ** (-0.5))
            kernels.gemm_bias_act(s, vt[f], out=o[f])
        out = self.to_out[0]
        return kernels.gemm_bias_residual(o.view(N, T, H, W, C), out.weight, out.bias, x, out=torch.empty_like(x))


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
        return _conv2d_run(self.conv, kernels.vae_upsample2x(x, False))


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
        x = self.mid_block(_conv2d_run(self.conv_in, z))
        for up in self.up_blocks:
            x = up(x)
        return _conv2d_run(self.conv_out, _gn(self.conv_norm_out, x))


class AutoencoderKL(nn.Module):
    """diffusers' AutoencoderKL, decoder half (``post_quant_conv``, ``decoder``).  The SDXL VAE of the released OpenSora
    v1.2 has block_out_channels (128, 256, 512, 512), layers_per_block 2, latent_channels 4."""

    def __init__(self, block_out_channels: Sequence[int] = (128, 256, 512, 512), layers_per_block: int = 2,
                 latent_channels: int = 4):
        super().__init__()
        self.config = type("Config", (), dict(block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                               latent_channels=latent_channels))()
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)
        self.decoder = SpatialDecoder(latent_channels, 3, block_out_channels, layers_per_block)
        self._pq = None

    def decode_frames(self, z):
        """z [N, 1, h, w, 16] -> [N, 1, 8h, 8w, 3]."""
        return self.decoder(kernels.gemm_bias_act(z, *self._pq))


class VideoAutoencoderKL(nn.Module):
    """Reference :488-555, decoder half: frames folded into the batch, ``micro_batch_size`` at a time."""

    def __init__(self, micro_batch_size: Optional[int] = 4, block_out_channels: Sequence[int] = (128, 256, 512, 512)):
        super().__init__()
        self.module = AutoencoderKL(block_out_channels)
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
            out[i:i + bs] = self.module.decode_frames(_pad_latent(x[i:i + bs] / SD_SCALING))
        return out.view(B, T, 8 * h, 8 * w, 3)


# =====================================================================================================================
# the pipeline
# =====================================================================================================================
class VideoAutoencoderPipeline(nn.Module):
    """OpenSora v1.2 VAE (reference :621-729 as built by OpenSoraVAE_V1_2 :731-761), decoder only: ``temporal_vae``
    (VAE_Temporal_SD) and ``spatial_vae.module`` (the SDXL AutoencoderKL), ``scale`` / ``shift`` buffers.

    ``spatial_block_out_channels`` narrows the image decoder (tests); every width must be one the GroupNorm kernels take
    (64, 128, 256, 512).  ``load_state_dict`` takes the checkpoint's full state dict: it drops ``*.encoder.*`` and
    ``*.quant_conv.*`` and is strict about every other key (``scale`` / ``shift`` may be absent: the released values stay).
    """

    def __init__(self, micro_frame_size: Optional[int] = 17, micro_batch_size: Optional[int] = 4,
                 spatial_block_out_channels: Sequence[int] = (128, 256, 512, 512), scale=SCALE, shift=SHIFT):
        super().__init__()
        bad = [c for c in spatial_block_out_channels if c not in _GN_CHANNELS]
        if bad or len(spatial_block_out_channels) < 1:
            raise ValueError(f"spatial_block_out_channels={tuple(spatial_block_out_channels)}: each width must be one of "
                             f"{_GN_CHANNELS}")
        self.spatial_vae = VideoAutoencoderKL(micro_batch_size, spatial_block_out_channels)
        self.temporal_vae = VAE_Temporal_SD()
        self.micro_frame_size = micro_frame_size
        self.micro_z_frame_size = self.temporal_vae.get_latent_size([micro_frame_size, None, None])[0] \
            if micro_frame_size is not None else None
        self.out_channels = self.temporal_vae.out_channels
        self.register_buffer("scale", torch.tensor(scale)[None, :, None, None, None])
        self.register_buffer("shift", torch.tensor(shift)[None, :, None, None, None])
        self._pack_key = None

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

    def load_state_dict(self, state_dict, strict: bool = True):
        kept = {k: v for k, v in state_dict.items() if not _dropped(k)}
        for k in ("scale", "shift"):
            if k not in kept:
                kept[k] = getattr(self, k)
        return super().load_state_dict(kept, strict=strict)

    @property
    def dtype(self):
        return self.temporal_vae.decoder.norm1.weight.dtype

    @property
    def device(self):
        return self.temporal_vae.decoder.norm1.weight.device

    def encode(self, x):
        raise NotImplementedError(f"{type(self).__name__}.encode: the VAE encoder is out of scope (decoder only)")

    # ---- kernel weights ----
    def _pack_weights(self):
        """Packs the weights for the kernels once per set of parameter tensors (after loading, .to(), ...)."""
        key = tuple((p.data_ptr(), p._version, p.dtype, p.device) for p in self.parameters())
        if key == self._pack_key:
            return
        for m in self.modules():
            if isinstance(m, CausalConv3d):
                m.pack()
            elif isinstance(m, nn.Conv2d) and m.kernel_size == (3, 3):
                _conv2d_pack(m)
            elif isinstance(m, nn.Conv2d) and m is not self.spatial_vae.module.post_quant_conv:  # 1x1 conv_shortcut
                m._w = m.weight.detach().flatten(1).contiguous()
            elif isinstance(m, Attention):
                m._w_qkv = torch.cat([m.to_q.weight, m.to_k.weight, m.to_v.weight]).detach().contiguous()
                m._b_qkv = torch.cat([m.to_q.bias, m.to_k.bias, m.to_v.bias]).detach().contiguous()
        pq = self.temporal_vae.post_quant_conv.conv
        self.temporal_vae._pq = _pad_1x1(pq.weight, pq.bias)
        pq = self.spatial_vae.module.post_quant_conv
        self.spatial_vae.module._pq = _pad_1x1(pq.weight, pq.bias)
        self._pack_key = key

    # ---- decoding ----
    @torch.no_grad()
    def decode(self, z, num_frames=None):
        """z [B, 4, T, h, w] -> video [B, 3, T', 8h, 8w] in [-1, 1]-ish (reference decode :672-695, cal_loss off)."""
        kernels.require_cuda(z, f"{type(self).__name__}.decode")
        z = z.to(self.dtype)
        kernels.require_cuda(z, f"{type(self).__name__}.decode", half_only=True)
        self._pack_weights()
        z = z * self.scale.to(z.dtype) + self.shift.to(z.dtype)
        zl = z.permute(0, 2, 3, 4, 1)  # [B, T, h, w, 4]
        if self.micro_frame_size is None:
            x_z = self.temporal_vae.decode(_pad_latent(zl), num_frames=num_frames)
        else:
            chunks = []
            for i in range(0, zl.shape[1], self.micro_z_frame_size):
                z_bs = _pad_latent(zl[:, i:i + self.micro_z_frame_size])
                chunks.append(self.temporal_vae.decode(z_bs, num_frames=min(self.micro_frame_size, num_frames)))
                num_frames -= self.micro_frame_size
            x_z = torch.cat(chunks, dim=1)
        return self.spatial_vae.decode(x_z).permute(0, 4, 1, 2, 3)


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
