"""Open-Sora-Plan v1.2.0 transformer (``OpenSoraT2V``) on the vsb200 sm_90a kernels (SURVEY.md section 8 row (f)4).

Reference: models/transformers/open_sora_plan_v120_transformer_3d.py -- model :1464-2112, ``BasicTransformerBlock`` :1092-1455,
``Attention`` + ``AttnProcessor2_0`` :647-960, ``RoPE3D`` / ``PositionGetter3D`` :39-118, ``PatchEmbed2D`` :245-369.  One stack
of blocks over ALL T*S tokens of a sample: ada_norm_single modulate -> full 3-D self-attention with RoPE3D (a third of
every head per axis, half-rotation inside each third) -> gate + residual -> text cross attention (padding mask = per-sample
key counts) + residual -> modulate -> tanh-GELU feed-forward -> gate + residual; PAB has the spatial and the cross gate and
caches the UN-gated attention output (:1352-1375, :1391-1416).

Kernels: every Linear = wgmma GEMM (q|k|v fused), ``vsb_ln_modulate`` (hidden 2304 = its 9-vector instantiation),
``vsb_gate_residual`` / ``vsb_residual_add``, ``vsb_qk_rope_halves`` (half = head_dim / 6, one table row per token) and
``vsb_attn_flash`` (csrc/attn_mma.cu, instantiated for head_dim 96).  Sequence parallelism as the reference (:907-916, :937-940, :1861-1866): the
tokens are split, self-attention exchanges tokens for heads (``comm.ulysses_*``), cross attention stays local.

State-dict compatible with the reference / HF ``LanguageBind/Open-Sora-Plan-v1.2.0`` transformers without a down-sampler
(``downsampler=None``: the released 29x480p / 93x480p ... "ROPE-L/122" models; the k33_s22 variants' depth-wise conv
attention down-sampler and conv feed-forward are not built).  Pinned against the reference file executed unmodified
(tests/test_oracle_vs_reference.py::test_osp_v120_*; diffusers leaves = the reference's vendored copies).
"""
import torch
import torch.nn as nn

from ... import kernels
from ...core.distributed import comm
from ...core.pab import pab_mgr
from ._attention import apply_rope_, cross_attention, packed_self_attention, ulysses_attention
from ._common import (AdaLNSingle, Lin2, PatchEmbed2D, ada_norm_single, ada_norm_single_out, fused_linear, grid_1d,
                      parallel_manager, pos_embed_2d, sincos_1d, text_lens)
from .latte_transformer_3d import _Attn, _FF


def rope3d_tables(head_dim, t, h, w, scales_thw, dtype, device):
    """cos / signed-sin tables [t*h*w, head_dim] of ``vsb_qk_rope_halves`` for RoPE3D (:63-118): axis a owns head_dim / 3
    channels, position / interpolation_scale_a (a float division), angles rounded to the compute dtype before cos / sin;
    tokens in cartesian_prod(t, y, x) order (:47-60).  The reference caches its cos / sin tables by (dim, length, device, dtype)
    WITHOUT the scale (:73-82): two axes of the same extent share the table of the first one (t, then h, then w) whatever
    their scales -- reproduced here."""
    Dax = head_dim // 3
    half = Dax // 2
    inv_freq = 1.0 / (10000.0 ** (torch.arange(0, Dax, 2).float() / Dax))
    pos = torch.cartesian_prod(torch.arange(t), torch.arange(h), torch.arange(w))  # [N, 3]
    sign = torch.cat([-torch.ones(half), torch.ones(half)])
    cs, sn, cache = [], [], {}
    for a, (n, sc) in enumerate(zip((t, h, w), scales_thw)):
        if n not in cache:
            tt = torch.arange(n, dtype=torch.float32) / sc
            freqs = torch.einsum("i,j->ij", tt, inv_freq).to(dtype)
            freqs = torch.cat((freqs, freqs), dim=-1)
            cache[n] = (freqs.cos().float(), freqs.sin().float())
        cs.append(cache[n][0][pos[:, a]])
        sn.append(cache[n][1][pos[:, a]] * sign)
    return torch.cat(cs, -1).contiguous().to(device), torch.cat(sn, -1).contiguous().to(device), half


class OSPBlock(nn.Module):
    def __init__(self, dim, cross_dim, bias=True):
        super().__init__()
        self.attn1 = _Attn(dim)
        self.attn2 = _Attn(dim, cross_dim)
        self.ff = _FF(dim)
        self.scale_shift_table = nn.Parameter(torch.randn(6, dim) / dim**0.5)
        self._fused = {}
        self.spatial_count = self.cross_count = 0
        self.spatial_last = self.cross_last = None


class OpenSoraT2V(nn.Module):
    def __init__(self, num_attention_heads=24, attention_head_dim=96, in_channels=4, out_channels=8, num_layers=32,
                 cross_attention_dim=2304, attention_bias=True, sample_size=(60, 80), sample_size_t=8, patch_size=2,
                 patch_size_t=1, activation_fn="gelu-approximate", norm_type="ada_norm_single", norm_elementwise_affine=False,
                 norm_eps=1e-6, caption_channels=4096, interpolation_scale_h=None, interpolation_scale_w=None,
                 interpolation_scale_t=None, attention_mode="xformers", downsampler=None, use_rope=True, **unused):
        super().__init__()
        if norm_type != "ada_norm_single" or activation_fn != "gelu-approximate" or norm_elementwise_affine or not attention_bias:
            raise NotImplementedError("vsb200 Open-Sora-Plan v1.2.0 implements the released configuration (ada_norm_single, tanh-GELU, biased projections)")
        if downsampler is not None:
            raise NotImplementedError("the conv down-sampled attention / conv feed-forward variants (downsampler != None) are not built")
        if patch_size_t != 1:
            raise NotImplementedError("patch_size_t != 1")
        if isinstance(sample_size, int):
            sample_size = (sample_size, sample_size)
        dim = num_attention_heads * attention_head_dim
        if use_rope and attention_head_dim % 6:
            raise ValueError("number of dimensions should be a multiple of three (and even per axis)")  # reference :105
        self.config = type("Cfg", (), dict(in_channels=in_channels, out_channels=out_channels, patch_size=patch_size,
                                           patch_size_t=patch_size_t, sample_size=tuple(sample_size), sample_size_t=sample_size_t,
                                           caption_channels=caption_channels, num_attention_heads=num_attention_heads,
                                           attention_head_dim=attention_head_dim, num_layers=num_layers, use_rope=use_rope,
                                           hidden_size=dim, cross_attention_dim=cross_attention_dim))()
        self.inner_dim, self.patch_size, self.out_channels, self.eps, self.use_rope = dim, patch_size, out_channels, norm_eps, use_rope
        st = ((sample_size_t - 1) // 16 + 1) if sample_size_t % 2 == 1 else sample_size_t / 16  # :1574-1583
        self.scale_t = interpolation_scale_t if interpolation_scale_t is not None else st
        self.scale_hw = (interpolation_scale_h if interpolation_scale_h is not None else sample_size[0] / 30,
                         interpolation_scale_w if interpolation_scale_w is not None else sample_size[1] / 40)
        self.pos_embed = PatchEmbed2D(patch_size, in_channels, dim)
        self._grid_hw = (sample_size[0] // patch_size, sample_size[1] // patch_size)
        self.num_frames = (sample_size_t - 1) // patch_size_t + 1 if sample_size_t % 2 == 1 else sample_size_t // patch_size_t
        if not use_rope:  # PatchEmbed2D(use_abs_pos=True) :270-283
            self.register_buffer("pos_table", pos_embed_2d(dim, self._grid_hw, self._grid_hw, self.scale_hw)[None], persistent=False)
            tpe = sincos_1d(dim, grid_1d(self.num_frames, self.num_frames, self.scale_t))
            self.register_buffer("temp_pos_embed", tpe.float()[None], persistent=False)
        self.transformer_blocks = nn.ModuleList([OSPBlock(dim, cross_attention_dim) for _ in range(num_layers)])
        self.scale_shift_table = nn.Parameter(torch.randn(2, dim) / dim**0.5)
        self.proj_out = nn.Linear(dim, patch_size_t * patch_size * patch_size * out_channels)
        self.adaln_single = AdaLNSingle(dim)
        self.caption_projection = Lin2(caption_channels, dim)  # PixArtAlphaTextProjection(act_fn='gelu_tanh')
        self._rope = {}
        self.parallel_manager = None

    @classmethod
    def from_pretrained(cls, path, subfolder: str = None, **config_overrides):
        """Reference pipeline_open_sora_plan.py:298-300 (``subfolder`` = "29x480p" ...), LOCAL directories."""
        from ...utils.checkpoint import build_from_pretrained

        return build_from_pretrained(cls, path, subfolder, **config_overrides)

    def enable_parallel(self, dp_size=None, sp_size=None, enable_cp=None):
        """Reference :1688-1700 (the forward never uses the cp group)."""
        self.parallel_manager = parallel_manager(dp_size, sp_size, enable_cp, self.config.num_attention_heads)

    def reset_pab_state(self):
        for b in self.transformer_blocks:
            b.spatial_count = b.cross_count = 0
            b.spatial_last = b.cross_last = None

    def _rope_for(self, T, h, w, dtype, device):
        key = (T, h, w, dtype, str(device))
        if key not in self._rope:
            self._rope[key] = rope3d_tables(self.config.attention_head_dim, T, h, w, (self.scale_t, *self.scale_hw), dtype, device)
        return self._rope[key]

    def _run_block(self, blk, x, enc2, mod, B, N, Ng, L, lens, rope, ts_int, sp_group):
        """x [B, N, C] (N = this rank's tokens, Ng = all tokens of a sample)."""
        K = kernels
        C, H = self.inner_dim, self.config.num_attention_heads
        D = C // H
        pab_on = pab_mgr.enable_pab()
        # ---- 3-D self attention ----
        reuse = False
        if pab_on:
            reuse, blk.spatial_count = pab_mgr.if_broadcast_spatial(ts_int, blk.spatial_count)
        if reuse:
            a = blk.spatial_last
        else:
            xm = K.ln_modulate(x, mod, None, 0, 1, B, 1, N, eps=self.eps)
            a1 = blk.attn1
            qkv = K.gemm_bias_act(xm.view(B * N, C), *fused_linear(blk._fused, a1.to_q, a1.to_k, a1.to_v))
            if sp_group is None:
                if rope is not None:
                    apply_rope_(qkv, rope, H, D, pos_div=1, pos_mod=N)
                o = packed_self_attention(qkv, B, N, H, D, D**-0.5)
            else:  # tokens for heads (:907-911): every token, H / sp heads; RoPE on the full sequence; back (:937-940)
                o = ulysses_attention(qkv.view(B, N, 3, H, D), 0, Ng, sp_group, D**-0.5, rope=rope)
            a = K.gemm_bias_act(o.view(B * N, C), blk.attn1.to_out[0].weight, blk.attn1.to_out[0].bias)
            if pab_on:
                blk.spatial_last = a
        K.gate_residual(x, a.view(B, N, C), mod, None, 2, B, 1, N, out=x)
        # ---- text cross attention (un-normalised input for ada_norm_single, :1396) ----
        reuse = False
        if pab_on:
            reuse, blk.cross_count = pab_mgr.if_broadcast_cross(ts_int, blk.cross_count)
        if reuse:
            xc = blk.cross_last
        else:
            a2 = blk.attn2
            q = K.gemm_bias_act(x.view(B * N, C), a2.to_q.weight, a2.to_q.bias)
            kv = K.gemm_bias_act(enc2, *fused_linear(blk._fused, a2.to_k, a2.to_v)).view(-1, 2, C)
            o = cross_attention(q, kv, B, N, L, H, D, D**-0.5, kv_lens=lens)
            xc = K.gemm_bias_act(o.view(B * N, C), a2.to_out[0].weight, a2.to_out[0].bias)
            if pab_on:
                blk.cross_last = xc
        K.residual_add(x, xc.view(B, N, C), out=x)
        # ---- feed-forward ----
        xm = K.ln_modulate(x, mod, None, 3, 4, B, 1, N, eps=self.eps)
        hdn = K.gemm_bias_act(xm.view(B * N, C), blk.ff.net[0].proj.weight, blk.ff.net[0].proj.bias, act=1)
        y = K.gemm_bias_act(hdn, blk.ff.net[2].weight, blk.ff.net[2].bias)
        K.gate_residual(x, y.view(B, N, C), mod, None, 5, B, 1, N, out=x)

    @torch.no_grad()
    def forward(self, hidden_states, timestep=None, encoder_hidden_states=None, added_cond_kwargs=None, class_labels=None,
                cross_attention_kwargs=None, attention_mask=None, encoder_attention_mask=None, use_image_num: int = 0,
                return_dict: bool = True, ts_int=None, **kwargs):
        """hidden_states [B, C, F, H, W] latents, timestep [B], encoder_hidden_states [B, 1, L, caption_channels],
        encoder_attention_mask [B, 1, L] (reference :1734-1960)."""
        K = kernels
        K.require_cuda(hidden_states, "Open-Sora-Plan v1.2.0")
        if use_image_num:
            raise NotImplementedError("joint image training is outside the inference path")
        if attention_mask is not None and not bool(attention_mask.to(torch.bool).all()):
            raise NotImplementedError("videosys_b200: a latent attention mask with masked positions (the pipeline passes ones)")
        dt = self.proj_out.weight.dtype
        pm = self.parallel_manager
        sp_group = pm.sp_group if (pm is not None and pm.sp_size > 1) else None
        if encoder_hidden_states.ndim == 4:
            encoder_hidden_states = encoder_hidden_states[:, 0]
        B, Cin, Fr, Hh, Ww = hidden_states.shape
        p, C = self.patch_size, self.inner_dim
        h, w = Hh // p, Ww // p
        S = h * w
        L = encoder_hidden_states.shape[1]
        lens = text_lens(encoder_attention_mask, B, L)
        x = hidden_states.to(dt).permute(0, 2, 1, 3, 4).reshape(B * Fr, Cin, Hh, Ww)
        x = self.pos_embed.proj(x).flatten(2).transpose(1, 2)  # conv: cuDNN (glue, once per step); [B*F, S, C]
        if not self.use_rope:
            if Fr != self.num_frames:
                raise NotImplementedError  # reference :333-334
            pos = self.pos_table if (h, w) == self._grid_hw else pos_embed_2d(C, (h, w), self._grid_hw, self.scale_hw)[None].to(x.device)
            x = (x + pos.to(x.dtype)).to(dt).view(B, Fr, S, C)
            x = (x + self.temp_pos_embed.to(dt).unsqueeze(2)).to(dt)
        x = x.reshape(B, Fr * S, C).contiguous()
        embedded, t6, enc = ada_norm_single(self.adaln_single, self.caption_projection, timestep, encoder_hidden_states, dt)
        enc2 = enc.reshape(B * L, C).contiguous()
        if pab_mgr.enable_pab() and ts_int is None:
            ts_int = int(timestep[0])
        rope = self._rope_for(Fr, h, w, dt, hidden_states.device) if self.use_rope else None
        Ng = Fr * S
        if sp_group is not None:  # reference :1861-1866 (no padding: the token count must divide)
            x = comm.split_sequence(x, sp_group, dim=1).contiguous()
        N = x.shape[1]
        for blk in self.transformer_blocks:
            mod = K.modulation_table(blk.scale_shift_table, t6, None)
            self._run_block(blk, x, enc2, mod, B, N, Ng, L, lens, rope, ts_int, sp_group)
        y = ada_norm_single_out(self.scale_shift_table, embedded, x, B, 1, N, 1e-6)
        y = K.gemm_bias_act(y.view(B * N, C), self.proj_out.weight, self.proj_out.bias).view(B, N, -1)
        if sp_group is not None:  # the head is row-wise: gather its narrow output (the reference gathers the C-wide rows, :1944-1948)
            y = comm.gather_sequence(y, sp_group, dim=1)
        Co = self.out_channels
        y = y.reshape(B, Fr, h, w, 1, p, p, Co)
        out = torch.einsum("nthwopqc->nctohpwq", y).reshape(B, Co, Fr, h * p, w * p)
        return (out,) if not return_dict else type("Out", (), {"sample": out})()
