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
import inspect
import os
from typing import Optional, Tuple

import torch
import torch.nn as nn

from ... import kernels

_GN_CHANNELS = (64, 128, 256, 512)  # channel counts vsb_vae_groupnorm_stats takes
_LATENT_PAD = 16  # latent channels are zero padded to this (the convolution's smallest Cin)


def _cast_tuple(t, length=1):
    return tuple(t) if isinstance(t, (tuple, list)) else (t,) * length


def _norm(c):
    """Normalize (reference :150-151 / :1179-1180)."""
    return nn.GroupNorm(num_groups=32, num_channels=c, eps=1e-6, affine=True)


def _gn(norm, x, out=None, t_off=0, act=True):
    stats = kernels.vae_groupnorm_stats(x, norm.num_groups, norm.eps)
    return kernels.vae_groupnorm_act(x, stats, norm.weight, norm.bias, out=out, t_off=t_off, act=act)


class CausalConv3d(nn.Module):
    """Reference CausalConv3d: kt - 1 copies of frame 0 first, spatial zero padding, bias always present."""

    def __init__(self, chan_in, chan_out, kernel_size, padding=0, stride=1):
        super().__init__()
        self.kernel_size = _cast_tuple(kernel_size, 3)
        self.time_kernel_size = self.kernel_size[0]
        self.chan_in, self.chan_out = chan_in, chan_out
        padding = list(_cast_tuple(padding, 3))
        padding[0] = 0
        self.conv = nn.Conv3d(chan_in, chan_out, self.kernel_size, stride=stride, padding=tuple(padding))
        self._w = None

    @property
    def weight(self):
        return self.conv.weight

    @property
    def bias(self):
        return self.conv.bias

    def input_buffer(self, x_shape, dtype, device):
        """[B, kt - 1 + T, H, W, Cin] for an input [B, T, H, W, Cin]: frames kt - 1 .. are the convolution's input."""
        B, T, H, W, C = x_shape
        return torch.empty(B, self.time_kernel_size - 1 + T, H, W, C, dtype=dtype, device=device)

    def run(self, buf, resid=None):
        kt = self.time_kernel_size
        if kt > 1:
            buf[:, :kt - 1] = buf[:, kt - 1:kt]
        return kernels.vae_conv3d(buf, self._w, self.bias, self.chan_out, kt, resid=resid, round_conv=True)


class Conv2d(nn.Conv2d):
    """v1.2.0 Conv2d (:116-147): a per-frame 3x3 convolution, i.e. kt = 1."""

    time_kernel_size = 1

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=0, **kw):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding)
        self.chan_in, self.chan_out = in_channels, out_channels
        self._w = None

    input_buffer = CausalConv3d.input_buffer
    run = CausalConv3d.run


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
        _gn(self.norm1, x, buf, t_off=2)
        h = self.conv1.run(buf)
        buf = self.conv2.input_buffer(h.shape, h.dtype, h.device)
        _gn(self.norm2, h, buf, t_off=2)
        if self.in_channels != self.out_channels:
            x = kernels.gemm_bias_act(x, self.nin_shortcut._w, self.nin_shortcut.bias)
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

    def forward(self, x):
        B, T, H, W, C = x.shape
        qkv = kernels.gemm_bias_act(_gn(self.norm, x, act=False), self._w_qkv, self._b_qkv)
        q, k, vt = kernels.vae_attn_split(qkv, C, self.mixed)
        P, Pp = H * W, k.shape[1]
        o = torch.empty(B * T, P, C, dtype=x.dtype, device=x.device)
        s = torch.empty(P, Pp, dtype=x.dtype, device=x.device)  # one frame's scores at a time
        for f in range(B * T):
            kernels.gemm_bias_act(q[f], k[f], out=s)
            kernels.vae_attn_softmax_(s, P, int(C) ** (-0.5))
            kernels.gemm_bias_act(s, vt[f], out=o[f])
        o = kernels.vae_attn_merge(o, B, T, H, W) if self.mixed else o.view(B, T, H, W, C)
        return kernels.gemm_bias_residual(o, self.proj_out._w, self.proj_out.bias, x, out=torch.empty_like(x))


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
        _gn(self.norm_out, h, buf, t_off=self.conv_out.time_kernel_size - 1)
        return self.conv_out.run(buf)


class _CausalVAEDecoderModel(nn.Module):
    """The decoder half of CausalVAEModel, shared by both versions.  ``load_state_dict`` takes the reference's full state
    dict: it drops ``encoder.*``, ``quant_conv.*`` and ``loss.*`` and is strict about every other key."""

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
        for m in mult:
            if cfg["hidden_size"] * m not in _GN_CHANNELS:
                raise ValueError(f"hidden_size={cfg['hidden_size']} x hidden_size_mult {mult}: each width must be one of {_GN_CHANNELS}")
        for k in ("z_channels", "embed_dim"):
            if not 0 < cfg[k] <= _LATENT_PAD:
                raise ValueError(f"{k}={cfg[k]}: the decoder pads the latent to {_LATENT_PAD} channels (need 1 .. 16)")
        self.use_quant_layer = use_quant_layer
        self.decoder = Decoder(cfg["z_channels"], cfg["hidden_size"], mult, cfg["decoder_conv_in"], cfg["decoder_conv_out"],
                               cfg["decoder_attention"], cfg["decoder_resnet_blocks"], cfg["decoder_spatial_upsample"],
                               cfg["decoder_temporal_upsample"], cfg["decoder_mid_resnet"], cfg["num_res_blocks"])
        if use_quant_layer:
            self.post_quant_conv = CausalConv3d(cfg["embed_dim"], cfg["z_channels"], 1)
        self.use_tiling = False
        self._pack_key = None

    # ---- loading ----
    @classmethod
    def from_config(cls, cfg: dict):
        keys = set(inspect.signature(cls.__init__).parameters) - {"self"}
        return cls(**{k: v for k, v in cfg.items() if k in keys})

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

    def load_state_dict(self, state_dict, strict: bool = True):
        kept = {k: v for k, v in state_dict.items() if not k.startswith(self._DROPPED_PREFIXES)}
        return super().load_state_dict(kept, strict=strict)

    @property
    def dtype(self):
        return self.decoder.norm_out.weight.dtype

    def enable_tiling(self, use_tiling: bool = True):
        self.use_tiling = use_tiling

    def disable_tiling(self):
        self.enable_tiling(False)

    def encode(self, x):
        raise NotImplementedError(f"{type(self).__name__}.encode: the VAE encoder is out of scope (decoder only)")

    # ---- kernel weights ----
    def _pack_weights(self):
        """Packs the weights for the kernels once per set of parameter tensors (after loading, .to(), ...)."""
        key = tuple((p.data_ptr(), p._version, p.dtype, p.device) for p in self.parameters())
        if key == self._pack_key:
            return
        for m in self.modules():
            if isinstance(m, (CausalConv3d, Conv2d)):
                w = m.weight.detach()
                m._w = kernels.pack_conv_weight(w) if w.shape[-1] == 3 else w.flatten(1).contiguous()
            elif isinstance(m, AttnBlock3DFix):
                m._w_qkv = torch.cat([m.q.weight, m.k.weight, m.v.weight]).flatten(1).detach().contiguous()
                m._b_qkv = torch.cat([m.q.bias, m.k.bias, m.v.bias]).detach().contiguous()
            elif isinstance(m, TimeUpsampleRes2x):
                alpha = torch.sigmoid(m.mix_factor.detach())
                m._alpha = (float(alpha), float(1 - alpha))
        if self.use_quant_layer:
            pq = self.post_quant_conv
            w = torch.zeros(_LATENT_PAD, _LATENT_PAD, dtype=pq.weight.dtype, device=pq.weight.device)
            w[:pq.chan_out, :pq.chan_in] = pq.weight.detach().flatten(1)
            b = torch.zeros(_LATENT_PAD, dtype=pq.weight.dtype, device=pq.weight.device)
            b[:pq.chan_out] = pq.bias.detach()
            self._pq = (w, b)
        self._pack_key = key

    # ---- decoding ----
    def _decode_tile(self, z):
        """post_quant_conv + decoder of z [B, Cz, T, h, w] -> [B, 3, T', 8h, 8w] (reference decode without tiling)."""
        B, Cz, T, h, w = z.shape
        zp = torch.zeros(B, T, h, w, _LATENT_PAD, dtype=z.dtype, device=z.device)
        zp[..., :Cz] = z.permute(0, 2, 3, 4, 1)
        if self.use_quant_layer:
            zp = kernels.gemm_bias_act(zp, *self._pq)
        return self.decoder(zp).permute(0, 4, 1, 2, 3)

    @torch.no_grad()
    def decode(self, z):
        """z [B, embed_dim, T, h, w] -> [B, 3, T', 8h, 8w] (the reference's CausalVAEModel.decode)."""
        kernels.require_cuda(z, f"{type(self).__name__}.decode")
        z = z.to(self.dtype)
        kernels.require_cuda(z, f"{type(self).__name__}.decode", half_only=True)
        self._pack_weights()
        if self.use_tiling and (z.shape[-1] > self.tile_latent_min_size or z.shape[-2] > self.tile_latent_min_size
                                or z.shape[-3] > self.tile_latent_min_size_t):
            return self.tiled_decode(z)
        return self._decode_tile(z)

    def blend_v(self, a, b, blend_extent: int):
        blend_extent = min(a.shape[3], b.shape[3], blend_extent)
        for y in range(blend_extent):
            b[:, :, :, y, :] = a[:, :, :, -blend_extent + y, :] * (1 - y / blend_extent) + b[:, :, :, y, :] * (y / blend_extent)
        return b

    def blend_h(self, a, b, blend_extent: int):
        blend_extent = min(a.shape[4], b.shape[4], blend_extent)
        for x in range(blend_extent):
            b[:, :, :, :, x] = a[:, :, :, :, -blend_extent + x] * (1 - x / blend_extent) + b[:, :, :, :, x] * (x / blend_extent)
        return b

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
        overlap_size = int(self.tile_latent_min_size * (1 - self.tile_overlap_factor))
        blend_extent = int(self.tile_sample_min_size * self.tile_overlap_factor)
        row_limit = self.tile_sample_min_size - blend_extent
        rows = []
        for i in range(0, z.shape[3], overlap_size):
            row = []
            for j in range(0, z.shape[4], overlap_size):
                tile = z[:, :, :, i:i + self.tile_latent_min_size, j:j + self.tile_latent_min_size]
                row.append(self._decode_tile(tile))
            rows.append(row)
        result_rows = []
        for i, row in enumerate(rows):
            result_row = []
            for j, tile in enumerate(row):
                if i > 0:
                    tile = self.blend_v(rows[i - 1][j], tile, blend_extent)
                if j > 0:
                    tile = self.blend_h(row[j - 1], tile, blend_extent)
                result_row.append(tile[:, :, :, :row_limit, :row_limit])
            result_rows.append(torch.cat(result_row, dim=4))
        return torch.cat(result_rows, dim=3)


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
        from ...utils.checkpoint import load_local_checkpoint

        cfg, sd = load_local_checkpoint(path, subfolder or "")
        vae = cls.from_config(cfg)
        vae.load_state_dict(sd)
        return vae


def decoder_class(version: str):
    """The decoder class of an Open-Sora-Plan version ("v110" / "v120")."""
    return {"v110": CausalVAEModelV110, "v120": CausalVAEModelV120}[version]
