"""Host-side building blocks shared by the CogVideoX, Open-Sora-Plan and OpenSora v1.2 VAE decoders: GroupNorm, the
causal convolution's weight packing / input buffer / launch, the single-head per-frame attention, latent padding, the
2-D tiling with blended seams, and the decoder-only model base (loading filter, weight-pack cache, ``decode`` preamble).

Activations are channels-last ``[B, T, H, W, C]``.  A convolution with kt time taps reads a buffer ``[B, kt - 1 + T, H,
W, Cin]`` whose first kt - 1 frames are its causal context; how those frames are filled differs between the reference
models (copies of frame 0, zeros, or the conv cache carried from the previous frame batch) and stays with each model.
"""
import inspect

import torch
import torch.nn as nn

from ... import kernels

GN_CHANNELS = (64, 128, 256, 512)  # channel counts vsb_vae_groupnorm_stats takes
LATENT_PAD = 16  # latent channels are zero padded to this (the convolution's smallest Cin)


def check_widths(widths, what):
    """Raises ValueError unless ``widths`` is non-empty and each is a channel count the GroupNorm kernels take."""
    if not widths or any(c not in GN_CHANNELS for c in widths):
        raise ValueError(f"{what}: each width must be one of {GN_CHANNELS}")


def _cast_tuple(t, length=1):
    return tuple(t) if isinstance(t, (tuple, list)) else (t,) * length


def group_norm(norm, x, out=None, t_off=0, *, act):
    """``norm`` (an nn.GroupNorm) of x, then ``act`` (False: none, True: x * sigmoid(x), 2: F.silu), into frames t_off..
    of ``out`` when given."""
    stats = kernels.vae_groupnorm_stats(x, norm.num_groups, norm.eps)
    return kernels.vae_groupnorm_act(x, stats, norm.weight, norm.bias, out=out, t_off=t_off, act=act)


# ---- convolutions: any nn.Conv2d (kt = 1, per frame) or nn.Conv3d (kt = kernel_size[0]) ----
def conv_kt(conv):
    return conv.kernel_size[0] if isinstance(conv, nn.Conv3d) else 1


def pack_conv(conv):
    """Sets ``conv._w`` / ``conv._b``: a 3x3 or (kt, 1, 1) weight in the layout of vae_conv3d / vae_conv_time, a 1x1
    (1x1x1) weight as a [Cout, Cin] GEMM weight.  A bias-free convolution carries a zero bias: 16-bit(conv + 0) is the
    rounded convolution."""
    w = conv.weight.detach()
    conv._w = w.flatten(1).contiguous() if all(k == 1 for k in w.shape[2:]) else kernels.pack_conv_weight(w)
    conv._b = conv.bias.detach() if conv.bias is not None else torch.zeros(conv.out_channels, dtype=w.dtype, device=w.device)


def conv_buffer(conv, x_shape, dtype, device):
    """[B, kt - 1 + T, H, W, C] for an input of shape [B, T, H, W, C]: frames kt - 1 .. are the convolution's input, the
    frames before them its causal context (left for the caller to fill)."""
    B, T, H, W, C = x_shape
    return torch.empty(B, conv_kt(conv) - 1 + T, H, W, C, dtype=dtype, device=device)


def run_conv(conv, buf, resid=None):
    """vae_conv3d of a conv_buffer (context frames filled) -> [B, T, H, W, Cout], + resid in the epilogue."""
    return kernels.vae_conv3d(buf, conv._w, conv._b, conv.out_channels, conv_kt(conv), resid=resid)


# ---- attention ----
def frame_attention(qkv, C, mixed):
    """softmax(Q K^T C^-0.5) V over each frame's H * W pixels of qkv [B, T, H, W, 3C] (single head, head dim C) ->
    [B, T, H, W, C]: one frame's scores materialised at a time, as the references compute them.  ``mixed`` reads and
    writes the frames as AttnBlock3D does (reshape of b c t h w to (b*t, c, h*w))."""
    B, T, H, W, _ = qkv.shape
    q, k, vt = kernels.vae_attn_split(qkv, C, mixed)
    P, Pp = H * W, k.shape[1]
    o = torch.empty(B * T, P, C, dtype=qkv.dtype, device=qkv.device)
    s = torch.empty(P, Pp, dtype=qkv.dtype, device=qkv.device)
    for f in range(B * T):
        kernels.gemm_bias_act(q[f], k[f], out=s)
        kernels.vae_attn_softmax_(s, P, int(C) ** (-0.5))
        kernels.gemm_bias_act(s, vt[f], out=o[f])
    return kernels.vae_attn_merge(o, B, T, H, W) if mixed else o.view(B, T, H, W, C)


def attention(x, norm, w_qkv, b_qkv, w_out, b_out, mixed):
    """The mid-block attention of x [B, T, H, W, C]: GroupNorm, q | k | v as one GEMM, frame_attention, and the output
    projection with the residual x in the GEMM epilogue."""
    qkv = kernels.gemm_bias_act(group_norm(norm, x, act=False), w_qkv, b_qkv)
    o = frame_attention(qkv, x.shape[-1], mixed)
    return kernels.gemm_bias_residual(o, w_out, b_out, x, out=torch.empty_like(x))


# ---- the latent ----
def pad_latent(z):
    """[..., c] (c <= 16) -> [..., 16], zero channels after c: the smallest Cin the convolution and the GEMM take."""
    zp = torch.zeros(*z.shape[:-1], LATENT_PAD, dtype=z.dtype, device=z.device)
    zp[..., :z.shape[-1]] = z
    return zp


def pad_1x1(weight, bias):
    """A c -> c' 1x1 convolution (c, c' <= 16) as a [16, 16] GEMM weight and a [16] bias (zero rows / columns)."""
    cout, cin = weight.shape[:2]
    w = torch.zeros(LATENT_PAD, LATENT_PAD, dtype=weight.dtype, device=weight.device)
    w[:cout, :cin] = weight.detach().flatten(1)
    b = torch.zeros(LATENT_PAD, dtype=weight.dtype, device=weight.device)
    b[:cout] = bias.detach()
    return w, b


# ---- tiling ----
def blend_v(a, b, blend_extent: int):
    blend_extent = min(a.shape[3], b.shape[3], blend_extent)
    for y in range(blend_extent):
        b[:, :, :, y, :] = a[:, :, :, -blend_extent + y, :] * (1 - y / blend_extent) + b[:, :, :, y, :] * (y / blend_extent)
    return b


def blend_h(a, b, blend_extent: int):
    blend_extent = min(a.shape[4], b.shape[4], blend_extent)
    for x in range(blend_extent):
        b[:, :, :, :, x] = a[:, :, :, :, -blend_extent + x] * (1 - x / blend_extent) + b[:, :, :, :, x] * (x / blend_extent)
    return b


def tiled_decode_2d(z, decode_tile, tile_latent_hw, tile_sample_hw, overlap_hw):
    """decode_tile over overlapping spatial tiles of z [B, C, T, h, w], with the reference's integer arithmetic: a tile
    of tile_latent_hw latent pixels starts every (1 - overlap) of a tile; each decoded tile's leading rows / columns are
    blended with the tile above / to its left, and its first tile_sample - blend_extent rows / columns are kept."""
    (lh, lw), (sh, sw), (oh, ow) = tile_latent_hw, tile_sample_hw, overlap_hw
    blend_height, blend_width = int(sh * oh), int(sw * ow)
    row_limit_height, row_limit_width = sh - blend_height, sw - blend_width
    rows = [[decode_tile(z[:, :, :, i:i + lh, j:j + lw]) for j in range(0, z.shape[4], int(lw * (1 - ow)))]
            for i in range(0, z.shape[3], int(lh * (1 - oh)))]
    result_rows = []
    for i, row in enumerate(rows):
        result_row = []
        for j, tile in enumerate(row):
            if i > 0:
                tile = blend_v(rows[i - 1][j], tile, blend_height)
            if j > 0:
                tile = blend_h(row[j - 1], tile, blend_width)
            result_row.append(tile[:, :, :, :row_limit_height, :row_limit_width])
        result_rows.append(torch.cat(result_row, dim=4))
    return torch.cat(result_rows, dim=3)


# ---- the top-level models ----
class DecoderOnlyVAE(nn.Module):
    """Base of the top-level decoder-only VAE models.  ``load_state_dict`` takes the reference's full state dict: it
    drops the keys ``_dropped`` names (the encoder side) and is strict about every other key."""

    _DROPPED_PREFIXES = ()

    def __init__(self):
        super().__init__()
        self._pack_key = None

    @classmethod
    def from_config(cls, cfg: dict):
        """The model of a config dict; keys the constructor does not take are ignored."""
        keys = set(inspect.signature(cls.__init__).parameters) - {"self"}
        return cls(**{k: v for k, v in cfg.items() if k in keys})

    @classmethod
    def _from_local_diffusers(cls, path: str, subfolder: str):
        """A local diffusers-style snapshot: ``config.json`` and the weights of ``path`` / ``subfolder``."""
        from ...utils.checkpoint import load_local_checkpoint

        cfg, sd = load_local_checkpoint(path, subfolder)
        vae = cls.from_config(cfg)
        vae.load_state_dict(sd)
        return vae

    def _dropped(self, key: str) -> bool:
        return key.startswith(self._DROPPED_PREFIXES)

    def load_state_dict(self, state_dict, strict: bool = True):
        kept = {k: v for k, v in state_dict.items() if not self._dropped(k)}
        return super().load_state_dict(kept, strict=strict)

    def encode(self, x, *args, **kwargs):
        raise NotImplementedError(f"{type(self).__name__}.encode: the VAE encoder is out of scope (decoder only)")

    def _pack_weights(self):
        """Packs the weights for the kernels once per set of parameter tensors (after loading, .to(), ...): every
        convolution (pack_conv), and every module with a ``pack()`` (the model's own included) packs the fused or padded
        weights it consumes."""
        key = tuple((p.data_ptr(), p._version, p.dtype, p.device) for p in self.parameters())
        if key == self._pack_key:
            return
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.Conv3d)):
                pack_conv(m)
            elif hasattr(m, "pack"):
                m.pack()
        self._pack_key = key

    def _decode_input(self, z):
        """decode's preamble: z on the GPU, cast to the parameter dtype (which must be 16-bit), the weights packed."""
        what = f"{type(self).__name__}.decode"
        kernels.require_cuda(z, what)
        z = z.to(self.dtype)
        kernels.require_cuda(z, what, half_only=True)
        self._pack_weights()
        return z
