"""Conditioning and bookkeeping code the model front ends share: the diffusers position / timestep embeddings restated
from their published semantics (diffusers==0.30.0), the process-mesh set-up, the fused projection weights, and the
PixArt-alpha ``ada_norm_single`` embedders and output modulation of Latte and Open-Sora-Plan."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import kernels
from ...core.distributed.parallel_mgr import ParallelManager


# ---- sin-cos embeddings ---------------------------------------------------------------------------------------------------
def timestep_sinusoid(timesteps: torch.Tensor, dim: int = 256, flip_sin_to_cos: bool = True, freq_shift: float = 0) -> torch.Tensor:
    """diffusers Timesteps(dim, flip_sin_to_cos, downscale_freq_shift): fp32 [cos | sin] ([sin | cos] unflipped)."""
    half = dim // 2
    exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=timesteps.device) / (half - freq_shift)
    emb = timesteps[:, None].float() * exponent.exp()[None]
    return torch.cat([emb.cos(), emb.sin()] if flip_sin_to_cos else [emb.sin(), emb.cos()], dim=-1)


def sincos_1d(embed_dim: int, pos: torch.Tensor) -> torch.Tensor:
    """get_1d_sincos_pos_embed_from_grid: [sin(pos w) | cos(pos w)], w_i = 10000^(-i / (embed_dim/2)), float64."""
    omega = 1.0 / 10000 ** (torch.arange(embed_dim // 2, dtype=torch.float64) / (embed_dim / 2.0))
    out = pos.reshape(-1).double()[:, None] * omega[None]
    return torch.cat([out.sin(), out.cos()], dim=1)


def grid_1d(n, base, scale):
    """Positions 0 .. n-1 rescaled to a base extent and divided by the interpolation scale."""
    return torch.arange(n, dtype=torch.float32) / (n / base) / scale


def pos_embed_2d(embed_dim, hw, base_hw, scale_hw):
    """get_2d_sincos_pos_embed: [h*w, embed_dim] float32.  np.meshgrid(grid_w, grid_h) puts w first, so the first half
    of the channels encodes the w coordinate, the second half h."""
    grid_w, grid_h = torch.meshgrid(grid_1d(hw[1], base_hw[1], scale_hw[1]), grid_1d(hw[0], base_hw[0], scale_hw[0]),
                                    indexing="xy")
    return torch.cat([sincos_1d(embed_dim // 2, grid_w), sincos_1d(embed_dim // 2, grid_h)], dim=1).float()


# ---- host bookkeeping -----------------------------------------------------------------------------------------------------
def text_lens(mask, B, L):
    """encoder_attention_mask [B, L] or [B, 1, L] (1 = keep) -> valid key counts per sample (None: every key); the kernel
    masks a suffix."""
    if mask is None:
        return None
    m = mask.reshape(B, -1)[:, -L:].to(torch.bool).cpu()
    lens = m.sum(-1)
    if not torch.equal(m, torch.arange(L)[None] < lens[:, None]):
        raise NotImplementedError("videosys_b200: the text mask must keep a prefix of the tokens (tokenizer padding)")
    if int(lens.min()) == 0:
        raise NotImplementedError("videosys_b200: a sample with no valid text token")
    return [int(v) for v in lens]


def parallel_manager(dp_size, sp_size, enable_cp, num_heads=None):
    """The reference's enable_parallel: CFG parallelism takes a factor 2 out of an even sp_size when ``enable_cp``.
    num_heads: head-scatter sequence parallelism needs the heads to divide among the sp ranks."""
    dp_size, sp_size = dp_size or 1, sp_size or 1
    cp_size = 1
    if enable_cp and sp_size % 2 == 0:
        sp_size, cp_size = sp_size // 2, 2
    if num_heads is not None and num_heads % sp_size:
        raise ValueError(f"Number of heads {num_heads} must be divisible by sequence parallel size {sp_size}")
    return ParallelManager(dp_size, cp_size, sp_size)


def fused_linear(cache: dict, *linears):
    """One [sum N, K] weight and bias for Linear layers that read the same input, kept in ``cache`` and rebuilt when a
    parameter changes (load_state_dict / .to())."""
    key = tuple(id(m) for m in linears)
    ver = tuple((p.data_ptr(), p._version, p.dtype) for m in linears for p in (m.weight, m.bias))
    hit = cache.get(key)
    if hit is None or hit[0] != ver:
        hit = cache[key] = (ver, torch.cat([m.weight for m in linears], 0).contiguous(),
                            torch.cat([m.bias for m in linears], 0).contiguous())
    return hit[1], hit[2]


# ---- PixArt-alpha ada_norm_single (Latte, Open-Sora-Plan) -----------------------------------------------------------------
class Lin2(nn.Module):
    """linear_1 -> activation -> linear_2 (TimestepEmbedding, PixArtAlphaTextProjection)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.linear_1 = nn.Linear(cin, cout)
        self.linear_2 = nn.Linear(cout, cout)


class _CombinedEmb(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.timestep_embedder = Lin2(256, dim)


class AdaLNSingle(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.emb = _CombinedEmb(dim)
        self.linear = nn.Linear(dim, 6 * dim)


class PatchEmbed2D(nn.Module):
    def __init__(self, patch, cin, dim):
        super().__init__()
        self.proj = nn.Conv2d(cin, dim, kernel_size=(patch, patch), stride=patch, bias=True)


def ada_norm_single(adaln: AdaLNSingle, caption: Lin2, timestep, captions, dt):
    """AdaLayerNormSingle (SiLU MLP on the 256-wide sinusoid, then the 6C block table rows) and the tanh-GELU caption
    projection.  Returns (embedded [B, C], t6 [B, 6C], text tokens [B, L, C])."""
    K = kernels
    te = adaln.emb.timestep_embedder
    t_emb = timestep_sinusoid(timestep).to(dt)
    embedded = K.gemm_bias_act(F.silu(K.gemm_bias_act(t_emb, te.linear_1.weight, te.linear_1.bias)), te.linear_2.weight,
                               te.linear_2.bias)
    t6 = K.gemm_bias_act(F.silu(embedded), adaln.linear.weight, adaln.linear.bias)
    enc = K.gemm_bias_act(K.gemm_bias_act(captions.to(dt).contiguous(), caption.linear_1.weight, caption.linear_1.bias, act=1),
                          caption.linear_2.weight, caption.linear_2.bias)
    return embedded, t6, enc


def ada_norm_single_out(table, embedded, x, B, T, S, eps):
    """The output head's modulation: LayerNorm (no affine) * (1 + scale) + shift, (shift, scale) = table [2, C] +
    embedded, on x viewed as [B, T, S, C]."""
    C = table.shape[1]
    tab6 = torch.cat([table, table.new_zeros(4, C)], 0)  # the modulate kernel addresses [2, B, 6, C] tables
    mod = kernels.modulation_table(tab6, torch.cat([embedded, embedded, embedded.new_zeros(B, 4 * C)], 1).contiguous(), None)
    return kernels.ln_modulate(x, mod, None, 0, 1, B, T, S, eps=eps)


def patch_embed_frames(embed: PatchEmbed2D, latent, pos, p, dt):
    """Tokens [B, F, S, C] of a latent [B, Cin, F, H, W]: every frame through the p x p patch convolution, plus the position
    table pos [1, S, C].  One kernel (vsb_patch_embed) for 16-tap embeddings; the cuDNN convolution otherwise."""
    proj = embed.proj
    x = kernels.patch_embed(latent.to(dt).contiguous(), proj.weight, proj.bias, pos[0].to(dt).contiguous(), p, p)
    if x is None:
        B, Cin, Fr, H, W = latent.shape
        x = latent.to(dt).permute(0, 2, 1, 3, 4).reshape(B * Fr, Cin, H, W)
        x = proj(x).flatten(2).transpose(1, 2)
        x = (x + pos.to(dt)).reshape(B, Fr, (H // p) * (W // p), proj.out_channels)
    return x
