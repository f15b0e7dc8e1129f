"""Open-Sora-Plan v1.1.0 transformer (the reference's second ``LatteT2V``) on the vsb200 sm_90a kernels (SURVEY.md section 8
row (f)4).

Reference: models/transformers/open_sora_plan_v110_transformer_3d.py -- model :2123-2790, spatial block
``BasicTransformerBlock`` :1734-2072, temporal block ``BasicTransformerBlock_`` :1370-1733, attention processor
:1125-1268, RoPE2D / RoPE1D with linear scaling :136-252, PatchEmbed :361-426, AdaLayerNormSingle :2074-2108,
CaptionProjection :340-358.  The block structure is Latte's (alternating spatial / temporal blocks, ada_norm_single, text
cross attention in the spatial blocks, PAB incl. the MLP skip): the block loop is ``LatteBlockStack`` (latte_transformer_3d.py
of this package) with two additions that exist only here:

  * half-rotation RoPE on q and k of ``attn1`` (``use_rope``): 2-D over the (y, x) patch position in the spatial blocks
    (each half of the head for one axis), 1-D over the frame index in the temporal blocks, linear position scaling with its
    integer truncation (:187-196, :244-252); ``vsb_qk_rope_halves`` in place on the packed qkv, tables built exactly as the
    reference builds its 16-bit cos / sin (angles rounded to the compute dtype before the cos: :149-152);
  * the text padding mask (:2440-2444, a -10000 bias on padded keys) as per-sample key counts of ``vsb_attn_flash``;
  * KV compression (``compress_kv_factor`` = k > 1, only without RoPE: :2200): the second-half blocks (d >= num_layers // 2,
    :2283-2320) carry ``attn1.sr`` (depth-wise Conv2d k x k / Conv1d k, stride k) and ``attn1.norm`` (LayerNorm, eps 1e-5);
    their keys and values come from norm(sr(tokens)) over the patch grid of each frame (spatial) or the frames of each patch
    after k - 1 copies of frame 0 when the frame count is odd (temporal), :1181-1197 -- ``vsb_kv_compress``, then the
    k | v GEMM on the compressed rows and ``vsb_attn_flash`` with fewer keys than queries.  The compressed latent mask
    (:2497) is all ones, as every mask this front end accepts.

State-dict compatible with the reference / HF ``LanguageBind/Open-Sora-Plan-v1.1.0`` transformer.  Not built: joint image
training (``use_image_num``), non-trivial latent
attention masks (the pipeline passes all-ones, pipeline_open_sora_plan.py:1119).  The diffusers leaf classes the
reference file imports (GELU, Timesteps, TimestepEmbedding) are restated from their published semantics.
"""
import torch
import torch.nn as nn

from ... import kernels
from ...core.distributed import comm
from ...core.pab import pab_mgr
from ._common import (AdaLNSingle, Lin2, PatchEmbed2D, ada_norm_single, ada_norm_single_out, parallel_manager,
                      patch_embed_frames, pos_embed_2d, sincos_1d, text_lens)
from .latte_transformer_3d import LatteBlockStack


class _CaptionProjection(Lin2):
    """reference :340-358 (linear_1 -> tanh-GELU -> linear_2; the unused y_embedding buffer is part of the state dict)."""

    def __init__(self, cin, dim, num_tokens=120):
        super().__init__(cin, dim)
        self.register_buffer("y_embedding", torch.randn(num_tokens, cin) / cin**0.5)


def rope_tables(head_dim: int, axes_pos, scale: float, dtype, device):
    """cos / signed-sin tables [n_tokens, head_dim] (fp32 copies of the reference's 16-bit values) of ``vsb_qk_rope_halves``.
    axes_pos: one LongTensor [n_tokens] per position axis (2-D: y, x; 1-D: t); every axis owns head_dim / len(axes)
    channels.  Reference RoPE2D / RoPE1D.get_cos_sin (:143-154, :207-217) with LinearScaling (:187-196): positions are
    divided by the factor and cast back to integers, the angle table is rounded to the compute dtype before cos / sin."""
    Dax = head_dim // len(axes_pos)
    half = Dax // 2
    pos = [(p.float() / scale).to(torch.long) for p in axes_pos]
    n = max(int(p.max()) for p in pos) + 1
    inv_freq = 1.0 / (10000.0 ** (torch.arange(0, Dax, 2).float() / Dax))
    freqs = torch.einsum("i,j->ij", torch.arange(n, dtype=torch.float32), inv_freq).to(dtype)
    freqs = torch.cat((freqs, freqs), dim=-1)
    cos, sin = freqs.cos().float(), freqs.sin().float()  # 16-bit values, widened
    sign = torch.cat([-torch.ones(half), torch.ones(half)])
    c = torch.cat([cos[p] for p in pos], dim=-1)
    s = torch.cat([sin[p] * sign for p in pos], dim=-1)
    return c.contiguous().to(device), s.contiguous().to(device), half


class LatteT2V(nn.Module):
    def __init__(self, num_attention_heads=16, patch_size_t=1, attention_head_dim=72, in_channels=4, out_channels=8,
                 num_layers=28, cross_attention_dim=1152, attention_bias=True, sample_size=(64, 64), patch_size=2,
                 activation_fn="gelu-approximate", norm_type="ada_norm_single", norm_elementwise_affine=False, norm_eps=1e-6,
                 caption_channels=4096, video_length=17, attention_mode="xformers", use_rope=True, model_max_length=300,
                 rope_scaling_type="linear", compress_kv_factor=1, interpolation_scale_1d=None, **unused):
        super().__init__()
        if norm_type != "ada_norm_single" or activation_fn != "gelu-approximate" or norm_elementwise_affine:
            raise NotImplementedError("vsb200 Open-Sora-Plan v1.1.0 implements the released configuration (ada_norm_single, tanh-GELU)")
        if int(compress_kv_factor) != compress_kv_factor or compress_kv_factor < 1:
            raise ValueError(f"compress_kv_factor must be a positive integer, got {compress_kv_factor}")
        if compress_kv_factor != 1 and use_rope:  # reference :2200
            raise ValueError("KV compression (compress_kv_factor > 1) and RoPE cannot both be enabled")
        if rope_scaling_type != "linear":
            raise ValueError(f"Unknown RoPE scaling type {rope_scaling_type}")  # reference :1150
        if isinstance(sample_size, int):
            sample_size = (sample_size, sample_size)
        dim = num_attention_heads * attention_head_dim
        self.config = type("Cfg", (), dict(in_channels=in_channels, out_channels=out_channels, patch_size=patch_size,
                                           sample_size=tuple(sample_size), video_length=video_length,
                                           caption_channels=caption_channels, num_attention_heads=num_attention_heads,
                                           attention_head_dim=attention_head_dim, num_layers=num_layers, use_rope=use_rope,
                                           hidden_size=model_max_length))()
        self.inner_dim, self.patch_size, self.out_channels, self.eps = dim, patch_size, out_channels, norm_eps
        self.use_rope, self.video_length = use_rope, video_length
        self.scale_2d = max(sample_size[0] // 64, 1)  # :2218-2219
        if interpolation_scale_1d is None:  # :2240-2247
            interpolation_scale_1d = (video_length - 1) // 16 if video_length % 2 == 1 else video_length // 16
        self.scale_1d = max(interpolation_scale_1d, 1)
        self.pos_embed = PatchEmbed2D(patch_size, in_channels, dim)
        gh, gw = sample_size[0] // patch_size, sample_size[1] // patch_size
        g = int((gh * gw) ** 0.5)  # reference PatchEmbed :387-389: a square table of int(sqrt(num_patches))
        self._grid = (gh, gw)
        self.register_buffer("pos_table", self._pos_2d(g, g)[None], persistent=False)
        self.adaln_single = AdaLNSingle(dim)
        self.caption_projection = _CaptionProjection(caption_channels, dim)
        stack = LatteBlockStack(dim, num_attention_heads, num_layers)
        self.transformer_blocks = stack.transformer_blocks
        self.temporal_transformer_blocks = stack.temporal_transformer_blocks
        self.compress_kv_factor = k = int(compress_kv_factor)
        if k != 1:  # second-half blocks, spatial and temporal (:2283-2320); layers and init as _init_compress (:1101-1122)
            for d in range(num_layers // 2, num_layers):
                for blk, sr in ((self.transformer_blocks[d], nn.Conv2d(dim, dim, k, stride=k, groups=dim)),
                                (self.temporal_transformer_blocks[d], nn.Conv1d(dim, dim, k, stride=k, groups=dim))):
                    sr.weight.data.fill_(1 / k ** (sr.weight.ndim - 2))
                    sr.bias.data.zero_()
                    blk.attn1.sr = sr
                    blk.attn1.norm = nn.LayerNorm(dim)
        self._stack = [stack]
        self.scale_shift_table = nn.Parameter(torch.randn(2, dim) / dim**0.5)
        self.proj_out = nn.Linear(dim, patch_size * patch_size * out_channels)
        tpe = sincos_1d(dim, torch.arange(0, video_length).unsqueeze(1) / self.scale_1d)  # :109-112
        self.register_buffer("temp_pos_embed", tpe.float()[None], persistent=False)
        self._rope = {}
        self.parallel_manager = None

    @classmethod
    def from_pretrained(cls, path, subfolder: str = None, **config_overrides):
        """Reference pipeline_open_sora_plan.py:294-296 (``subfolder`` = "65x512x512" / "221x512x512"), LOCAL directories."""
        from ...utils.checkpoint import build_from_pretrained

        return build_from_pretrained(cls, path, subfolder, **config_overrides)

    def enable_parallel(self, dp_size=None, sp_size=None, enable_cp=None):
        """Reference :2344-2356."""
        self.parallel_manager = parallel_manager(dp_size, sp_size, enable_cp)

    def reset_pab_state(self):
        self._stack[0].reset_pab_state()

    def _rope_for(self, Fr, h, w, dtype, device):
        key = (Fr, h, w, dtype, str(device))
        if key not in self._rope:
            D = self.config.attention_head_dim
            yx = torch.cartesian_prod(torch.arange(h), torch.arange(w))  # PositionGetter2D :262-268
            self._rope[key] = {"spatial": rope_tables(D, [yx[:, 0], yx[:, 1]], self.scale_2d, dtype, device),
                               "temporal": rope_tables(D, [torch.arange(Fr)], self.scale_1d, dtype, device)}
        return self._rope[key]

    def _pos_2d(self, h, w):
        """reference get_2d_sincos_pos_embed :75-106: both axes divided by (extent / grid height) and the 2-D scale."""
        base, s = self._grid[0], self.scale_2d
        return pos_embed_2d(self.inner_dim, (h, w), (base, base), (s, s))

    @torch.no_grad()
    def forward(self, hidden_states, timestep=None, all_timesteps=None, encoder_hidden_states=None, added_cond_kwargs=None,
                class_labels=None, cross_attention_kwargs=None, attention_mask=None, encoder_attention_mask=None,
                use_image_num: int = 0, enable_temporal_attentions: bool = True, return_dict: bool = True, ts_int=None):
        """hidden_states [B, C, F, H, W] latents, timestep [B], encoder_hidden_states [B, 1, L, caption_channels] (or
        [B, L, ...]), encoder_attention_mask [B, 1, L] / [B, L] (reference :2406-2790)."""
        K = kernels
        K.require_cuda(hidden_states, "Open-Sora-Plan v1.1.0")
        if use_image_num or not enable_temporal_attentions:
            raise NotImplementedError("joint image training / spatial-only mode are outside the inference path")
        if attention_mask is not None and not bool(attention_mask.to(torch.bool).all()):
            raise NotImplementedError("videosys_b200: a latent attention mask with masked positions (the pipeline passes ones)")
        dt = self.proj_out.weight.dtype
        pm = self.parallel_manager
        cpar = pm is not None and pm.cp_size > 1
        sp = pm is not None and pm.sp_size > 1
        if encoder_hidden_states.ndim == 4:
            encoder_hidden_states = encoder_hidden_states[:, 0]
        if cpar:  # reference :2456-2471
            hidden_states, timestep, encoder_hidden_states = (
                comm.split_sequence(v, pm.cp_group, dim=0) for v in (hidden_states, timestep, encoder_hidden_states))
            if encoder_attention_mask is not None:
                encoder_attention_mask = comm.split_sequence(encoder_attention_mask, pm.cp_group, dim=0)
        B, _, Fr, H, W = hidden_states.shape
        if Fr != self.video_length:
            raise ValueError(f"{Fr} latent frames, but the temporal position table has {self.video_length} (reference :2656)")
        p, C = self.patch_size, self.inner_dim
        h, w = H // p, W // p
        S = h * w
        L = encoder_hidden_states.shape[1]
        k = self.compress_kv_factor
        pad_t = k - 1 if Fr % 2 == 1 else 0  # the temporal compression prepends frame 0 for an odd frame count (:1190-1192)
        if k != 1 and (h < k or w < k or (Fr + pad_t) < k):
            raise ValueError(f"KV compression by {k} needs at least {k} patches per axis and {k} frames, got {h}x{w} patches and "
                             f"{Fr} frames (+{pad_t} padding)")
        lens = text_lens(encoder_attention_mask, B, L)
        if (h, w) == self._grid and S == self.pos_table.shape[1]:
            pos = self.pos_table
        else:  # reference PatchEmbed.forward :412-420
            pos = self._pos_2d(h, w)[None].to(hidden_states.device)
        x = patch_embed_frames(self.pos_embed, hidden_states, pos, p, dt)
        embedded, t6, enc = ada_norm_single(self.adaln_single, self.caption_projection, timestep, encoder_hidden_states, dt)
        if pab_mgr.enable_pab() and ts_int is None:
            ts_int = int(timestep[0])
        if all_timesteps is not None and torch.is_tensor(all_timesteps):
            all_timesteps = all_timesteps.tolist()
        rope = self._rope_for(Fr, h, w, dt, hidden_states.device) if self.use_rope else None
        tpe = self.temp_pos_embed  # added before the first temporal block, with or without RoPE (:2656)
        Fg = Fr
        if sp:  # reference :2529-2541
            comm.set_pad("temporal", Fr, pm.sp_group)
            comm.set_pad("spatial", S, pm.sp_group)
            x = comm.split_sequence(x, pm.sp_group, dim=1, pad=comm.get_pad("temporal"))
            tpe = comm.split_sequence(tpe, pm.sp_group, dim=1, pad=comm.get_pad("temporal"))
            Fr = x.shape[1]
        x = self._stack[0](x, enc, t6, tpe, ts_int=ts_int, all_timesteps=all_timesteps, sp_group=pm.sp_group if sp else None,
                           rope=rope, enc_lens=lens, kv_grid=(h, w), kv_pad_t=pad_t)
        y = ada_norm_single_out(self.scale_shift_table, embedded, x.view(B, Fr * S, C), B, Fr, S, self.eps)
        y = K.gemm_bias_act(y, self.proj_out.weight, self.proj_out.bias)  # [B, F*S, p*p*Cout]
        if sp:
            y = comm.gather_sequence(y.view(B, Fr, S, -1), pm.sp_group, dim=1, pad=comm.get_pad("temporal"))
            Fr = Fg
        Co = self.out_channels
        y = y.reshape(B * Fr, h, w, p, p, Co)
        y = torch.einsum("nhwpqc->nchpwq", y).reshape(B * Fr, Co, h * p, w * p)
        out = y.reshape(B, Fr, Co, h * p, w * p).permute(0, 2, 1, 3, 4).contiguous()
        if cpar:  # reference :2763-2764
            out = comm.gather_sequence(out, pm.cp_group, dim=0)
        return (out,) if not return_dict else type("Out", (), {"sample": out})()
