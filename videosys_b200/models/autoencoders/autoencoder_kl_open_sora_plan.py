"""Open-Sora-Plan causal-VAE decoder, v1.1.0 and v1.2.0 (mirror of videosys/models/autoencoders/
autoencoder_kl_open_sora_plan_v110.py: Decoder :251-354, CausalVAEModel :357-790, and the modules it names, :899-992,
:1117-1167, :1418-1450, :1510-1596; autoencoder_kl_open_sora_plan_v120.py: :40-151, :277-415, :467-502, Decoder :629-738,
CausalVAEModel :741-1078) on the sm_90a kernels of csrc/vae_conv.cu and csrc/vae_osp.cu.

Only the decoder is in scope: ``encode`` raises ``NotImplementedError``.  The modules keep the reference's parameter names
and shapes under ``decoder.*`` and ``post_quant_conv.*``.  Activations stay channels-last ``[B, T, H, W, C]`` between
kernels:
  - every causal convolution reads a buffer that holds its kt - 1 context frames (copies of frame 0, reference
    CausalConv3d.forward) and then the frames the previous kernel wrote there (GroupNorm + nonlinearity, the linear
    up-sampler);
  - the latent (4 channels) is padded with zero channels to 16, the smallest channel count the convolution takes, once per
    decoded tile; ``post_quant_conv`` and ``nin_shortcut`` (1x1x1) are GEMMs on the pixel rows;
  - the attention block runs q | k | v as one GEMM, S = Q K^T, the scaled softmax and O = P V per frame (materialised, as
    the reference computes it), and ``proj_out`` with the block residual in the GEMM epilogue.
``decode``, ``tiled_decode`` and ``tiled_decode2d`` reproduce the reference's integer arithmetic.
"""
import glob
import os
from typing import Optional, Tuple

import torch
import torch.nn as nn

from ... import kernels
from ._common import (LATENT_PAD, DecoderOnlyVAE, _cast_tuple, attention, check_widths, conv_buffer, group_norm, pad_1x1,
                      pad_latent, run_conv, tiled_decode_2d)


def _norm(c):
    """Normalize (reference :150-151 / :1179-1180)."""
    return nn.GroupNorm(num_groups=32, num_channels=c, eps=1e-6, affine=True)


class CausalConv3d(nn.Module):
    """Reference CausalConv3d: kt - 1 copies of frame 0 first, spatial zero padding, bias always present."""

    def __init__(self, chan_in, chan_out, kernel_size, padding=0, stride=1):
        super().__init__()
        self.kernel_size = _cast_tuple(kernel_size, 3)
        self.time_kernel_size = self.kernel_size[0]
        padding = list(_cast_tuple(padding, 3))
        padding[0] = 0
        self.conv = nn.Conv3d(chan_in, chan_out, self.kernel_size, stride=stride, padding=tuple(padding))

    def input_buffer(self, x_shape, dtype, device):
        return conv_buffer(self.conv, x_shape, dtype, device)

    def run(self, buf, resid=None):
        kt = self.time_kernel_size
        if kt > 1:
            buf[:, :kt - 1] = buf[:, kt - 1:kt]
        return run_conv(self.conv, buf, resid)


class Conv2d(nn.Conv2d):
    """v1.2.0 Conv2d (:116-147): a per-frame 3x3 convolution, i.e. kt = 1."""

    time_kernel_size = 1

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=0, **kw):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding)

    def input_buffer(self, x_shape, dtype, device):
        return conv_buffer(self, x_shape, dtype, device)

    def run(self, buf, resid=None):
        return run_conv(self, buf, resid)


class ResnetBlock3D(nn.Module):
    """v1.1.0 :1418-1450, v1.2.0 :277-315 (ResnetBlock3D_GC :467-502 has the same forward): norm1 + act -> conv1 ->
    norm2 + act -> conv2, + x (through nin_shortcut when the width changes) in conv2's epilogue."""

    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout=0.0):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = in_channels if out_channels is None else out_channels
        self.norm1 = _norm(in_channels)
        self.conv1 = CausalConv3d(in_channels, self.out_channels, 3, padding=1)
        self.norm2 = _norm(self.out_channels)
        self.conv2 = CausalConv3d(self.out_channels, self.out_channels, 3, padding=1)
        if self.in_channels != self.out_channels:
            self.nin_shortcut = CausalConv3d(in_channels, self.out_channels, 1, padding=0)

    def forward(self, x):
        buf = self.conv1.input_buffer(x.shape, x.dtype, x.device)
        group_norm(self.norm1, x, buf, t_off=2, act=True)
        h = self.conv1.run(buf)
        buf = self.conv2.input_buffer(h.shape, h.dtype, h.device)
        group_norm(self.norm2, h, buf, t_off=2, act=True)
        if self.in_channels != self.out_channels:
            x = kernels.gemm_bias_act(x, self.nin_shortcut.conv._w, self.nin_shortcut.conv._b)
        return self.conv2.run(buf, resid=x)


ResnetBlock3D_GC = ResnetBlock3D


class AttnBlock3DFix(nn.Module):
    """v1.2.0 :360-415 (also v1.1.0 :939-992): single-head attention over each frame's h*w pixels, head dim C."""

    mixed = False  # AttnBlock3D reads its frames through reshape(b*t, c, h*w) of b c t h w

    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = _norm(in_channels)
        self.q = CausalConv3d(in_channels, in_channels, kernel_size=1, stride=1)
        self.k = CausalConv3d(in_channels, in_channels, kernel_size=1, stride=1)
        self.v = CausalConv3d(in_channels, in_channels, kernel_size=1, stride=1)
        self.proj_out = CausalConv3d(in_channels, in_channels, kernel_size=1, stride=1)
        self._w_qkv = self._b_qkv = None

    def pack(self):
        qkv = [self.q.conv, self.k.conv, self.v.conv]
        self._w_qkv = torch.cat([c.weight for c in qkv]).flatten(1).detach().contiguous()
        self._b_qkv = torch.cat([c.bias for c in qkv]).detach().contiguous()

    def forward(self, x):
        out = self.proj_out.conv
        return attention(x, self.norm, self._w_qkv, self._b_qkv, out._w, out._b, self.mixed)


class AttnBlock3D(AttnBlock3DFix):
    """v1.1.0 :899-936, the v1.1.0 constructor default: equal to AttnBlock3DFix only for T = 1."""

    mixed = True


class SpatialUpsample2x(nn.Module):
    """v1.1.0 :1510-1530, v1.2.0 :318-341: nearest 2x in H and W per frame, then a (1, 3, 3) convolution."""

    def __init__(self, chan_in, chan_out, kernel_size=(3, 3), stride=(1, 1), unup=False):
        super().__init__()
        self.unup = unup
        self.conv = CausalConv3d(chan_in, chan_out, (1,) + tuple(kernel_size), stride=(1,) + tuple(stride), padding=1)

    def forward(self, x):
        u = x if self.unup else kernels.vae_upsample2x(x, False)
        return self.conv.run(u)


class Spatial2xTime2x3DUpsample(nn.Module):
    """v1.2.0 :344-357: trilinear (1, 2, 2) on frame 0 and (2, 2, 2) on frames 1.., then a causal 3x3x3 convolution."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.conv = CausalConv3d(in_channels, out_channels, kernel_size=3, padding=1)

    def forward(self, x):
        B, T, H, W, C = x.shape
        buf = self.conv.input_buffer((B, 2 * T - 1, 2 * H, 2 * W, C), x.dtype, x.device)
        kernels.vae_upsample_linear2x(x, True, True, out=buf, t_off=2)
        return self.conv.run(buf)


class TimeUpsample2x(nn.Module):
    """v1.1.0 :1545-1554: linear 2x along T on frames 1.."""

    def __init__(self, chan_in, chan_out):
        super().__init__()

    def forward(self, x):
        return kernels.vae_upsample_linear2x(x, False, True) if x.shape[1] > 1 else x


class TimeUpsampleRes2x(nn.Module):
    """v1.1.0 :1578-1596: alpha * up(x) + (1 - alpha) * conv(up(x)), alpha = sigmoid(mix_factor) in the parameter dtype."""

    def __init__(self, in_channels, out_channels, kernel_size=3, mix_factor=2.0):
        super().__init__()
        self.conv = CausalConv3d(in_channels, out_channels, kernel_size, padding=1)
        self.mix_factor = nn.Parameter(torch.Tensor([mix_factor]))
        self._alpha = None

    def pack(self):
        alpha = torch.sigmoid(self.mix_factor.detach())
        self._alpha = (float(alpha), float(1 - alpha))

    def forward(self, x):
        B, T, H, W, C = x.shape
        buf = self.conv.input_buffer((B, 2 * T - 1, H, W, C), x.dtype, x.device)
        kernels.vae_upsample_linear2x(x, False, True, out=buf, t_off=2)
        return kernels.vae_mix(buf, self.conv.run(buf), *self._alpha, t_off=2)


_CONVS = ("CausalConv3d", "Conv2d")
_RESNETS = ("ResnetBlock3D", "ResnetBlock3D_GC")
_MODULES = {c.__name__: c for c in (CausalConv3d, Conv2d, ResnetBlock3D, AttnBlock3DFix, AttnBlock3D, SpatialUpsample2x,
                                    Spatial2xTime2x3DUpsample, TimeUpsample2x, TimeUpsampleRes2x)}
_MODULES["ResnetBlock3D_GC"] = ResnetBlock3D


class Decoder(nn.Module):
    """v1.1.0 :251-354, v1.2.0 :629-738 (attn_resolutions empty: no attention inside the up levels)."""

    def __init__(self, z_channels, hidden_size, hidden_size_mult, conv_in, conv_out, attention, resnet_blocks,
                 spatial_upsample, temporal_upsample, mid_resnet, num_res_blocks):
        super().__init__()
        self.num_resolutions = len(hidden_size_mult)
        self.num_res_blocks = num_res_blocks
        block_in = hidden_size * hidden_size_mult[-1]
        self.conv_in = _MODULES[conv_in](z_channels, block_in, kernel_size=3, padding=1)
        self.mid = nn.Module()
        self.mid.block_1 = _MODULES[mid_resnet](in_channels=block_in, out_channels=block_in)
        self.mid.attn_1 = _MODULES[attention](block_in)
        self.mid.block_2 = _MODULES[mid_resnet](in_channels=block_in, out_channels=block_in)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block = nn.ModuleList()
            block_out = hidden_size * hidden_size_mult[i_level]
            for _ in range(num_res_blocks + 1):
                block.append(_MODULES[resnet_blocks[i_level]](in_channels=block_in, out_channels=block_out))
                block_in = block_out
            up = nn.Module()
            up.block = block
            up.attn = nn.ModuleList()
            if spatial_upsample[i_level]:
                up.upsample = _MODULES[spatial_upsample[i_level]](block_in, block_in)
            if temporal_upsample[i_level]:
                up.time_upsample = _MODULES[temporal_upsample[i_level]](block_in, block_in)
            self.up.insert(0, up)
        self.norm_out = _norm(block_in)
        self.conv_out = _MODULES[conv_out](block_in, 3, kernel_size=3, padding=1)

    def forward(self, z):
        """z [B, T, h, w, 16] (channels-last, zero padded) -> [B, T', 8h, 8w, 3]."""
        buf = self.conv_in.input_buffer(z.shape, z.dtype, z.device)
        buf[:, self.conv_in.time_kernel_size - 1:] = z
        h = self.conv_in.run(buf)
        h = self.mid.block_1(h)
        h = self.mid.attn_1(h)
        h = self.mid.block_2(h)
        for i_level in reversed(range(self.num_resolutions)):
            up = self.up[i_level]
            for b in up.block:
                h = b(h)
            if hasattr(up, "upsample"):
                h = up.upsample(h)
            if hasattr(up, "time_upsample"):
                h = up.time_upsample(h)
        buf = self.conv_out.input_buffer(h.shape, h.dtype, h.device)
        group_norm(self.norm_out, h, buf, t_off=self.conv_out.time_kernel_size - 1, act=True)
        return self.conv_out.run(buf)


class _CausalVAEDecoderModel(DecoderOnlyVAE):
    """The decoder half of CausalVAEModel, shared by both versions.  ``load_state_dict`` drops the ``encoder.*``,
    ``quant_conv.*`` and ``loss.*`` entries of the reference's full state dict."""

    _DROPPED_PREFIXES = ("encoder.", "quant_conv.", "loss.")
    _ACCEPTED = {}  # decoder slot -> accepted module names

    def _build(self, cfg, use_quant_layer):
        self.config = type("Config", (), cfg)()
        slots = {"conv_in": [cfg["decoder_conv_in"]], "conv_out": [cfg["decoder_conv_out"]],
                 "attention": [cfg["decoder_attention"]],
                 "resnet_blocks": list(cfg["decoder_resnet_blocks"]) + [cfg["decoder_mid_resnet"]],
                 "spatial_upsample": list(cfg["decoder_spatial_upsample"]),
                 "temporal_upsample": list(cfg["decoder_temporal_upsample"]), "q_conv": [cfg["q_conv"]]}
        for slot, names in slots.items():
            for n in names:
                if n not in self._ACCEPTED[slot]:
                    raise NotImplementedError(f"{type(self).__name__}: decoder module {n!r} ({slot}) is not supported; "
                                              f"accepted: {sorted(x for x in self._ACCEPTED[slot] if x)}")
        if list(cfg["attn_resolutions"]):
            raise NotImplementedError(f"attn_resolutions={cfg['attn_resolutions']!r}: attention inside the up levels "
                                      "(AttnBlock) is not supported")
        mult = tuple(cfg["hidden_size_mult"])
        if len(cfg["decoder_resnet_blocks"]) != len(mult) or len(cfg["decoder_spatial_upsample"]) != len(mult) or \
                len(cfg["decoder_temporal_upsample"]) != len(mult):
            raise ValueError("decoder_resnet_blocks / _spatial_upsample / _temporal_upsample need one entry per hidden_size_mult")
        check_widths([cfg["hidden_size"] * m for m in mult], f"hidden_size={cfg['hidden_size']} x hidden_size_mult {mult}")
        for k in ("z_channels", "embed_dim"):
            if not 0 < cfg[k] <= LATENT_PAD:
                raise ValueError(f"{k}={cfg[k]}: the decoder pads the latent to {LATENT_PAD} channels (need 1 .. 16)")
        self.use_quant_layer = use_quant_layer
        self.decoder = Decoder(cfg["z_channels"], cfg["hidden_size"], mult, cfg["decoder_conv_in"], cfg["decoder_conv_out"],
                               cfg["decoder_attention"], cfg["decoder_resnet_blocks"], cfg["decoder_spatial_upsample"],
                               cfg["decoder_temporal_upsample"], cfg["decoder_mid_resnet"], cfg["num_res_blocks"])
        if use_quant_layer:
            self.post_quant_conv = CausalConv3d(cfg["embed_dim"], cfg["z_channels"], 1)
        self.use_tiling = False

    # ---- loading ----
    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None):
        """A LOCAL directory (``path`` / ``subfolder``): its last ``*.ckpt`` with ``config.json`` next to it (the
        reference's VideoBaseAE.from_pretrained + init_from_ckpt); v1.1.0 also takes diffusers-style weights.  No hub."""
        import json

        d = os.path.join(path, subfolder) if subfolder else path
        ckpts = sorted(glob.glob(os.path.join(d, "*.ckpt")))
        if not ckpts:
            return cls._from_diffusers_weights(path, subfolder)
        with open(os.path.join(d, "config.json")) as f:
            vae = cls.from_config(json.load(f))
        vae.load_state_dict(vae.unwrap_checkpoint(torch.load(ckpts[-1], map_location="cpu", weights_only=True)))
        return vae

    @classmethod
    def _from_diffusers_weights(cls, path, subfolder):
        raise FileNotFoundError(f"{cls.__name__}.from_pretrained: no *.ckpt in {os.path.join(path, subfolder or '')} "
                                "(local directories only)")

    @property
    def dtype(self):
        return self.decoder.norm_out.weight.dtype

    def enable_tiling(self, use_tiling: bool = True):
        self.use_tiling = use_tiling

    def disable_tiling(self):
        self.enable_tiling(False)

    # ---- kernel weights ----
    def pack(self):
        if self.use_quant_layer:
            self._pq = pad_1x1(self.post_quant_conv.conv.weight, self.post_quant_conv.conv.bias)

    # ---- decoding ----
    def _decode_tile(self, z):
        """post_quant_conv + decoder of z [B, Cz, T, h, w] -> [B, 3, T', 8h, 8w] (reference decode without tiling)."""
        zp = pad_latent(z.permute(0, 2, 3, 4, 1))
        if self.use_quant_layer:
            zp = kernels.gemm_bias_act(zp, *self._pq)
        return self.decoder(zp).permute(0, 4, 1, 2, 3)

    @torch.no_grad()
    def decode(self, z):
        """z [B, embed_dim, T, h, w] -> [B, 3, T', 8h, 8w] (the reference's CausalVAEModel.decode)."""
        z = self._decode_input(z)
        if self.use_tiling and (z.shape[-1] > self.tile_latent_min_size or z.shape[-2] > self.tile_latent_min_size
                                or z.shape[-3] > self.tile_latent_min_size_t):
            return self.tiled_decode(z)
        return self._decode_tile(z)

    def tiled_decode(self, x):
        t = x.shape[2]
        t_chunk_idx = [i for i in range(0, t, self.tile_latent_min_size_t - 1)]
        if len(t_chunk_idx) == 1 and t_chunk_idx[0] == 0:
            t_chunk_start_end = [[0, t]]
        else:
            t_chunk_start_end = [[t_chunk_idx[i], t_chunk_idx[i + 1] + 1] for i in range(len(t_chunk_idx) - 1)]
            if t_chunk_start_end[-1][-1] > t:
                t_chunk_start_end[-1][-1] = t
            elif t_chunk_start_end[-1][-1] < t:
                t_chunk_start_end.append([t_chunk_idx[-1], t])
        dec_ = []
        for idx, (start, end) in enumerate(t_chunk_start_end):
            dec = self.tiled_decode2d(x[:, :, start:end])
            dec_.append(dec[:, :, 1:] if idx != 0 else dec)  # each later chunk repeats the previous chunk's last frame
        return torch.cat(dec_, dim=2)

    def tiled_decode2d(self, z):
        return tiled_decode_2d(z, lambda tile: self._decode_tile(tile), (self.tile_latent_min_size,) * 2,
                               (self.tile_sample_min_size,) * 2, (self.tile_overlap_factor,) * 2)


_V120_ACCEPTED = {"conv_in": _CONVS, "conv_out": _CONVS, "attention": ("AttnBlock3DFix",), "resnet_blocks": _RESNETS,
                  "spatial_upsample": ("", "SpatialUpsample2x", "Spatial2xTime2x3DUpsample"), "temporal_upsample": ("",),
                  "q_conv": ("CausalConv3d",)}
_V110_ACCEPTED = {"conv_in": ("CausalConv3d",), "conv_out": ("CausalConv3d",), "attention": ("AttnBlock3D", "AttnBlock3DFix"),
                  "resnet_blocks": ("ResnetBlock3D",), "spatial_upsample": ("", "SpatialUpsample2x"),
                  "temporal_upsample": ("", "TimeUpsample2x", "TimeUpsampleRes2x"), "q_conv": ("CausalConv3d",)}


class CausalVAEModelV120(_CausalVAEDecoderModel):
    """v1.2.0 CausalVAEModel (:741-1078), decoder only, with the reference's constructor keywords."""

    _ACCEPTED = _V120_ACCEPTED

    def __init__(self, hidden_size: int = 128, z_channels: int = 4, hidden_size_mult: Tuple[int] = (1, 2, 4, 4),
                 attn_resolutions: Tuple[int] = [], dropout: float = 0.0, resolution: int = 256, double_z: bool = True,
                 embed_dim: int = 4, num_res_blocks: int = 2, q_conv: str = "CausalConv3d",
                 encoder_conv_in="CausalConv3d", encoder_conv_out="CausalConv3d", encoder_attention="AttnBlock3D",
                 encoder_resnet_blocks=("ResnetBlock3D",) * 4,
                 encoder_spatial_downsample=("SpatialDownsample2x", "SpatialDownsample2x", "SpatialDownsample2x", ""),
                 encoder_temporal_downsample=("", "TimeDownsample2x", "TimeDownsample2x", ""),
                 encoder_mid_resnet="ResnetBlock3D", decoder_conv_in="CausalConv3d", decoder_conv_out="CausalConv3d",
                 decoder_attention="AttnBlock3D", decoder_resnet_blocks=("ResnetBlock3D",) * 4,
                 decoder_spatial_upsample=("", "SpatialUpsample2x", "SpatialUpsample2x", "SpatialUpsample2x"),
                 decoder_temporal_upsample=("", "", "TimeUpsample2x", "TimeUpsample2x"),
                 decoder_mid_resnet="ResnetBlock3D", use_quant_layer: bool = True):
        super().__init__()
        cfg = {k: v for k, v in locals().items() if k not in ("self", "__class__")}
        self._build(cfg, use_quant_layer)
        self.tile_sample_min_size = 256
        self.tile_sample_min_size_t = 33
        self.tile_latent_min_size = int(self.tile_sample_min_size / (2 ** (len(hidden_size_mult) - 1)))
        self.tile_latent_min_size_t = 16
        self.tile_overlap_factor = 0.125

    @staticmethod
    def unwrap_checkpoint(sd):
        """init_from_ckpt (:1051-1078): the EMA weights when present (unless NOT_USE_EMA_MODEL is set), else state_dict
        or its gen_model."""
        if "ema_state_dict" in sd and len(sd["ema_state_dict"]) > 0 and os.environ.get("NOT_USE_EMA_MODEL", 0) == 0:
            return {k.replace("module.", ""): v for k, v in sd["ema_state_dict"].items()}
        if "state_dict" in sd:
            return sd["state_dict"]["gen_model"] if "gen_model" in sd["state_dict"] else sd["state_dict"]
        return sd


class CausalVAEModelV110(_CausalVAEDecoderModel):
    """v1.1.0 CausalVAEModel (:357-790), decoder only, with the reference's constructor keywords."""

    _ACCEPTED = _V110_ACCEPTED

    def __init__(self, lr: float = 1e-5, hidden_size: int = 128, z_channels: int = 4, hidden_size_mult: Tuple[int] = (1, 2, 4, 4),
                 attn_resolutions: Tuple[int] = [], dropout: float = 0.0, resolution: int = 256, double_z: bool = True,
                 embed_dim: int = 4, num_res_blocks: int = 2,
                 loss_type: str = "opensora.models.ae.videobase.losses.LPIPSWithDiscriminator",
                 loss_params: dict = {"kl_weight": 0.000001, "logvar_init": 0.0, "disc_start": 2001, "disc_weight": 0.5},
                 q_conv: str = "CausalConv3d", encoder_conv_in: str = "CausalConv3d", encoder_conv_out: str = "CausalConv3d",
                 encoder_attention: str = "AttnBlock3D", encoder_resnet_blocks: Tuple[str] = ("ResnetBlock3D",) * 4,
                 encoder_spatial_downsample: Tuple[str] = ("SpatialDownsample2x", "SpatialDownsample2x", "SpatialDownsample2x", ""),
                 encoder_temporal_downsample: Tuple[str] = ("", "TimeDownsample2x", "TimeDownsample2x", ""),
                 encoder_mid_resnet: str = "ResnetBlock3D", decoder_conv_in: str = "CausalConv3d",
                 decoder_conv_out: str = "CausalConv3d", decoder_attention: str = "AttnBlock3D",
                 decoder_resnet_blocks: Tuple[str] = ("ResnetBlock3D",) * 4,
                 decoder_spatial_upsample: Tuple[str] = ("", "SpatialUpsample2x", "SpatialUpsample2x", "SpatialUpsample2x"),
                 decoder_temporal_upsample: Tuple[str] = ("", "", "TimeUpsample2x", "TimeUpsample2x"),
                 decoder_mid_resnet: str = "ResnetBlock3D"):
        super().__init__()
        cfg = {k: v for k, v in locals().items() if k not in ("self", "__class__")}
        self._build(cfg, True)
        self.tile_sample_min_size = 256
        self.tile_sample_min_size_t = 65
        self.tile_latent_min_size = int(self.tile_sample_min_size / (2 ** (len(hidden_size_mult) - 1)))
        t_down_ratio = [i for i in encoder_temporal_downsample if len(i) > 0]
        self.tile_latent_min_size_t = int((self.tile_sample_min_size_t - 1) / (2 ** len(t_down_ratio))) + 1
        self.tile_overlap_factor = 0.25

    @staticmethod
    def unwrap_checkpoint(sd):
        """init_from_ckpt (:779-790): the ``state_dict`` entry when present."""
        return sd["state_dict"] if "state_dict" in sd else sd

    @classmethod
    def _from_diffusers_weights(cls, path, subfolder):
        """Without a *.ckpt the reference falls back to ModelMixin.from_pretrained: config.json + diffusers weights."""
        return cls._from_local_diffusers(path, subfolder or "")


def decoder_class(version: str):
    """The decoder class of an Open-Sora-Plan version ("v110" / "v120")."""
    return {"v110": CausalVAEModelV110, "v120": CausalVAEModelV120}[version]
