"""Latte transformer blocks on the vsb200 sm_90a kernels (block level: SURVEY.md section 8 row a16).

``LatteBlockStack`` holds the parameters of LatteT2V's ``transformer_blocks`` / ``temporal_transformer_blocks`` under
the reference's state_dict names (diffusers ``Attention``: attn1/attn2.to_q|to_k|to_v|to_out.0, ``FeedForward``:
ff.net.0.proj / ff.net.2, ``scale_shift_table``; norms carry no parameters) and runs the block loop of
models/transformers/latte_transformer_3d.py:1312-1425 (inference, use_image_num = 0) on the same kernels as STDiT3:

  * activations stay token-major [B, F, S, C]; the reference's two rearranges per block pair are strides;
  * to_q / to_k / to_v are fused into one [3C, C] GEMM (weights concatenated once, lazily);
  * spatial self-attention = vsb_attn_flash on the packed qkv; temporal (F < 30) = vsb_attn_short with flags 3 (no q/k
    norm, SDPA rounding); cross attention = one kv GEMM per sample (the reference repeats the text per frame and
    recomputes it F times: latte_transformer_3d.py:1290-1296) + vsb_attn_flash.

``LatteT2V`` adds the embedders and the output head (reference :846-1470); the diffusers pieces (PatchEmbed's 2-D sincos
table, Timesteps / TimestepEmbedding inside PixArtAlphaCombinedTimestepSizeEmbeddings, PixArtAlphaTextProjection) are
restated from their published semantics (diffusers==0.30.0: parity unpinned for those, SURVEY.md 8c).  Compute dtype:
fp16 (the reference's, pipeline_latte.py:201) or bf16.  PAB: spatial / temporal / cross broadcast and the MLP skip.
"""
from typing import Optional

import torch
import torch.nn as nn

from ... import kernels
from ...core.distributed import comm
from ...core.pab import pab_mgr
from ._attention import (apply_rope_, cross_attention, packed_self_attention, temporal_attention,
                         temporal_cross_attention)
from ._common import (AdaLNSingle, Lin2, PatchEmbed2D, ada_norm_single, ada_norm_single_out, fused_linear, parallel_manager,
                      patch_embed_frames, pos_embed_2d, sincos_1d)


class _Attn(nn.Module):
    def __init__(self, dim, cross_dim=None):
        super().__init__()
        kv = cross_dim or dim
        self.to_q = nn.Linear(dim, dim, bias=True)
        self.to_k = nn.Linear(kv, dim, bias=True)
        self.to_v = nn.Linear(kv, dim, bias=True)
        self.to_out = nn.ModuleList([nn.Linear(dim, dim, bias=True), nn.Identity()])


class _GELUProj(nn.Module):
    def __init__(self, dim, inner):
        super().__init__()
        self.proj = nn.Linear(dim, inner)


class _FF(nn.Module):
    def __init__(self, dim, mult=4):
        super().__init__()
        self.net = nn.ModuleList([_GELUProj(dim, dim * mult), nn.Identity(), nn.Linear(dim * mult, dim)])


class LatteBlock(nn.Module):
    def __init__(self, dim, heads, temporal, block_idx=0):
        super().__init__()
        self.temporal = temporal
        self.block_idx = block_idx
        self.attn1 = _Attn(dim)
        if not temporal:
            self.attn2 = _Attn(dim, dim)
        self.ff = _FF(dim)
        self.scale_shift_table = nn.Parameter(torch.randn(6, dim) / dim**0.5)
        self._fused = {}
        self.reset_pab()

    def reset_pab(self):
        # reference attributes: spatial_count / count (temporal), cross_count, mlp_count; spatial_last / last_out, cross_last
        self.attn_count = self.cross_count = self.mlp_count = 0
        self.last_attn = self.last_cross = None


def _sr_taps(cache, sr):
    """sr.weight [C, 1, *window] as [taps, C] (tap-major), kept in ``cache`` and rebuilt when the parameter changes."""
    ver = (sr.weight.data_ptr(), sr.weight._version, sr.weight.dtype)
    hit = cache.get("sr")
    if hit is None or hit[0] != ver:
        hit = cache["sr"] = (ver, sr.weight.reshape(sr.weight.shape[0], -1).t().contiguous())
    return hit[1]


def _compressed_attention(blk, xm, B, Fr, S, grid, pad_t, H, D):
    """Self-attention of a block with Open-Sora-Plan v1.1.0's KV compression (open_sora_plan_v110_transformer_3d.py:1181-1197):
    queries from every modulated token xm [B*Fr*S, C], keys / values from attn1.norm(attn1.sr(xm)) -- a stride-k depth-wise
    conv over the (h, w) = grid patches of each frame (spatial block) or over the Fr frames of each patch after pad_t copies of
    frame 0 (temporal block).  Returns [B*Fr*S, C] in the order of xm."""
    a1, C = blk.attn1, H * D
    k = a1.sr.stride[0]
    q = kernels.gemm_bias_act(xm, a1.to_q.weight, a1.to_q.bias)
    taps = _sr_taps(blk._fused, a1.sr)
    if blk.temporal:  # Conv1d: ATen's native depthwise kernel (one rounding after the bias)
        xc = kernels.kv_compress(xm, taps, a1.sr.bias, a1.norm.weight, a1.norm.bias, B, Fr, S, 1, (k, 1, 1), pad_t, a1.norm.eps,
                                 round_conv=False)
    else:  # Conv2d on a channels-last view: cuDNN (the conv rounded, then the bias added)
        xc = kernels.kv_compress(xm, taps, a1.sr.bias, a1.norm.weight, a1.norm.bias, B, Fr, grid[0], grid[1], (1, k, k), 0,
                                 a1.norm.eps, round_conv=True)
    kv = kernels.gemm_bias_act(xc.view(-1, C), *fused_linear(blk._fused, a1.to_k, a1.to_v)).view(-1, 2, C)
    if blk.temporal:
        return temporal_cross_attention(q, kv, B, Fr, xc.shape[1], S, H, D, D**-0.5)
    return cross_attention(q, kv, B * Fr, S, xc.shape[2] * xc.shape[3], H, D, D**-0.5).view(-1, C)


class LatteBlockStack(nn.Module):
    def __init__(self, hidden_size=1152, num_heads=16, depth=28):
        super().__init__()
        self.hidden_size, self.num_heads, self.depth = hidden_size, num_heads, depth
        self.transformer_blocks = nn.ModuleList([LatteBlock(hidden_size, num_heads, False, i) for i in range(depth)])
        self.temporal_transformer_blocks = nn.ModuleList([LatteBlock(hidden_size, num_heads, True, i) for i in range(depth)])

    def reset_pab_state(self):
        for b in [*self.transformer_blocks, *self.temporal_transformer_blocks]:
            b.reset_pab()

    @torch.no_grad()
    def forward(self, x: torch.Tensor, enc: torch.Tensor, timestep6: torch.Tensor, temp_pos_embed: Optional[torch.Tensor] = None,
                ts_int: Optional[int] = None, all_timesteps=None, sp_group=None, rope: Optional[dict] = None, enc_lens=None,
                kv_grid=None, kv_pad_t: int = 0):
        """x [B, F, S, C] fp16 / bf16 (CUDA), enc [B, L, C], timestep6 [B, 6C]; returns [B, F, S, C].
        PAB (reference blocks :372-517, :700-824): ts_int = int(org_timestep[0]) on the host, all_timesteps = the
        scheduler's timestep list (python ints) for the MLP skip windows.
        sp_group: Latte's flavour of DSP (reference :734-745, :826-843): x (and temp_pos_embed) hold this rank's FRAMES;
        spatial blocks are local; a temporal block switches its modulated input to a patch shard with every frame for
        the attention (qkv, softmax, out projection) and switches the result back (pads: comm.get_pad).
        rope (Open-Sora-Plan v1.1.0, open_sora_plan_v110_transformer_3d.py:1217-1232): {"spatial": (cos, sin_signed, half),
        "temporal": (...)} tables of ``vsb_qk_rope_halves`` indexed by the token's patch / frame; enc_lens: valid text tokens per
        sample (the reference's -10000 bias on padded keys, :2440-2444).
        kv_grid / kv_pad_t (Open-Sora-Plan v1.1.0 KV compression, blocks whose attn1 has ``sr``): the (h, w) patch grid of a
        frame and the leading copies of frame 0 the temporal compression reads."""
        K = kernels
        K.require_cuda(x, "Latte / Open-Sora-Plan blocks", half_only=True)
        B, Fr, S, C = x.shape
        H = self.num_heads
        D = C // H
        L = enc.shape[1]
        x = x.contiguous().clone()
        enc2 = enc.reshape(B * L, C).contiguous()
        xf = x.view(B, Fr * S, C)
        pab_on = pab_mgr.enable_pab()
        if pab_on and ts_int is None:
            raise RuntimeError("PAB needs the host integer timestep (ts_int)")
        for i in range(self.depth):
            for blk in (self.transformer_blocks[i], self.temporal_transformer_blocks[i]):
                if blk.temporal and i == 0 and temp_pos_embed is not None:  # the caller passes it for F > 1 (:1391)
                    x.add_(temp_pos_embed.reshape(1, Fr, 1, C).to(x.dtype))  # glue op (once per forward)
                mod = K.modulation_table(blk.scale_shift_table, timestep6, None)
                # ---- self attention (spatial over S per frame / temporal over F per patch) ----
                reuse = False
                if pab_on:
                    gate = pab_mgr.if_broadcast_temporal if blk.temporal else pab_mgr.if_broadcast_spatial
                    reuse, blk.attn_count = gate(ts_int, blk.attn_count)
                if reuse:
                    K.residual_add(xf, blk.last_attn, out=xf)  # the cached value is the GATED output (:422-430)
                else:
                    xm = K.ln_modulate(xf, mod, None, 0, 1, B, Fr, S)
                    switch = blk.temporal and sp_group is not None
                    Ft, St = Fr, S  # extents the temporal attention sees
                    if switch:  # frame shard -> patch shard (scatter S, gather F)
                        xm = comm.all_to_all_with_pad(xm.view(B, Fr, S, C), sp_group, scatter_dim=2, gather_dim=1,
                                                      scatter_pad=comm.get_pad("spatial"),
                                                      gather_pad=comm.get_pad("temporal")).contiguous()
                        Ft, St = xm.shape[1], xm.shape[2]
                        xm = xm.view(B * Ft * St, C)
                    a1 = blk.attn1
                    if hasattr(a1, "sr"):  # Open-Sora-Plan v1.1.0 KV compression (only its second-half blocks have sr)
                        o = _compressed_attention(blk, xm, B, Ft, St, kv_grid, kv_pad_t, H, D)
                    else:
                        qkv = K.gemm_bias_act(xm, *fused_linear(blk._fused, a1.to_q, a1.to_k, a1.to_v))
                        if blk.temporal:
                            o = temporal_attention(qkv, B, Ft, St, H, D, D**-0.5, 32, sdpa=True,
                                                   rope=None if rope is None else rope["temporal"])
                        else:
                            if rope is not None:
                                apply_rope_(qkv, rope["spatial"], H, D, pos_div=1, pos_mod=S)
                            o = packed_self_attention(qkv, B * Fr, S, H, D, D**-0.5, short_max=29, sdpa=True)
                    y = K.gemm_bias_act(o.view(-1, C), blk.attn1.to_out[0].weight, blk.attn1.to_out[0].bias)
                    if switch:  # patch shard -> frame shard (scatter F, gather S)
                        y = comm.all_to_all_with_pad(y.view(B, Ft, St, C), sp_group, scatter_dim=1, gather_dim=2,
                                                     scatter_pad=comm.get_pad("temporal"),
                                                     gather_pad=comm.get_pad("spatial")).contiguous()
                    cache = None
                    if pab_on:
                        if blk.last_attn is None or blk.last_attn.shape != xf.shape:
                            blk.last_attn = torch.empty_like(xf)
                        cache = blk.last_attn
                    K.gate_residual(xf, y.view(B, Fr * S, C), mod, None, 2, B, Fr, S, out=xf, cache_out=cache)
                # ---- text cross attention (spatial blocks only) ----
                if not blk.temporal:
                    reuse = False
                    if pab_on:
                        reuse, blk.cross_count = pab_mgr.if_broadcast_cross(ts_int, blk.cross_count)
                    if reuse:
                        K.residual_add(xf, blk.last_cross, out=xf)
                    else:
                        a2 = blk.attn2
                        q = K.gemm_bias_act(xf, a2.to_q.weight, a2.to_q.bias)
                        kv = K.gemm_bias_act(enc2, *fused_linear(blk._fused, a2.to_k, a2.to_v)).view(-1, 2, C)
                        o = cross_attention(q, kv, B, Fr * S, L, H, D, D**-0.5, kv_lens=enc_lens)
                        out = blk.last_cross if (pab_on and blk.last_cross is not None and blk.last_cross.shape == xf.shape) else None
                        xc = K.gemm_bias_act(o, a2.to_out[0].weight, a2.to_out[0].bias, out=out)
                        if pab_on:
                            blk.last_cross = xc
                        K.residual_add(xf, xc.view(B, Fr * S, C), out=xf)
                # ---- feed-forward, with the PAB MLP skip (Latte enables it: pipeline_latte.py:48-61) ----
                skip = keep = False
                rng = None
                if pab_on:
                    skip, cnt, keep, rng = pab_mgr.if_broadcast_mlp(ts_int, blk.mlp_count, blk.block_idx, all_timesteps, blk.temporal)
                    if cnt is not None:
                        blk.mlp_count = cnt
                if skip:
                    ff = pab_mgr.get_mlp_output(rng, ts_int, blk.block_idx, blk.temporal)  # stored GATED output
                    K.residual_add(xf, ff, out=xf)
                else:
                    xm = K.ln_modulate(xf, mod, None, 3, 4, B, Fr, S)
                    h = K.gemm_bias_act(xm, blk.ff.net[0].proj.weight, blk.ff.net[0].proj.bias, act=1)
                    y = K.gemm_bias_act(h, blk.ff.net[2].weight, blk.ff.net[2].bias)
                    ffc = torch.empty_like(xf) if keep else None
                    K.gate_residual(xf, y, mod, None, 5, B, Fr, S, out=xf, cache_out=ffc)
                    if keep:
                        pab_mgr.save_mlp_output(ts_int, blk.block_idx, ffc, blk.temporal)
        return x


# ---- the whole denoiser (reference LatteT2V :846-1470, ada_norm_single / PixArt-alpha conditioning) ------------------------
class LatteT2V(nn.Module):
    """State-dict compatible with the reference / HF ``maxin-cn/Latte-1`` transformer (same parameter names), forward on the
    vsb200 kernels.  ``enable_parallel`` as the reference (:1127-1139): frame-sharded DSP (temporal blocks switch to a
    patch shard and back) and CFG parallelism."""

    def __init__(self, num_attention_heads=16, attention_head_dim=72, in_channels=4, out_channels=8, num_layers=28,
                 cross_attention_dim=1152, attention_bias=True, sample_size=64, patch_size=2, activation_fn="gelu-approximate",
                 norm_type="ada_norm_single", norm_elementwise_affine=False, norm_eps=1e-6, caption_channels=4096,
                 video_length=16, **unused):
        super().__init__()
        if norm_type != "ada_norm_single" or activation_fn != "gelu-approximate" or norm_elementwise_affine:
            raise NotImplementedError("vsb200 LatteT2V implements the Latte-1 configuration (ada_norm_single, tanh-GELU)")
        if sample_size == 128:
            raise NotImplementedError("resolution / aspect-ratio micro-conditions (sample_size 128) are not built")
        dim = num_attention_heads * attention_head_dim
        self.config = type("Cfg", (), dict(in_channels=in_channels, out_channels=out_channels, patch_size=patch_size,
                                           sample_size=sample_size, video_length=video_length, caption_channels=caption_channels,
                                           num_attention_heads=num_attention_heads, attention_head_dim=attention_head_dim,
                                           num_layers=num_layers))()
        self.inner_dim, self.patch_size, self.out_channels, self.eps = dim, patch_size, out_channels, norm_eps
        self.pos_embed = PatchEmbed2D(patch_size, in_channels, dim)
        grid = sample_size // patch_size
        self.register_buffer("pos_table", self._pos_2d(grid, grid)[None], persistent=False)
        self.adaln_single = AdaLNSingle(dim)
        self.caption_projection = Lin2(caption_channels, dim)
        stack = LatteBlockStack(dim, num_attention_heads, num_layers)
        self.transformer_blocks = stack.transformer_blocks
        self.temporal_transformer_blocks = stack.temporal_transformer_blocks
        self._stack = [stack]
        self.scale_shift_table = nn.Parameter(torch.randn(2, dim) / dim**0.5)
        self.proj_out = nn.Linear(dim, patch_size * patch_size * out_channels)
        self.register_buffer("temp_pos_embed", sincos_1d(dim, torch.arange(video_length).float()).float()[None], persistent=False)
        self.parallel_manager = None

    @classmethod
    def from_pretrained(cls, path, subfolder: str = "transformer", **config_overrides):
        """Reference pipeline_latte.py:196-199 (``video_length=16``), for a LOCAL snapshot directory."""
        from ...utils.checkpoint import build_from_pretrained

        return build_from_pretrained(cls, path, subfolder, **config_overrides)

    def enable_parallel(self, dp_size=None, sp_size=None, enable_cp=None):
        """Reference :1127-1139."""
        self.parallel_manager = parallel_manager(dp_size, sp_size, enable_cp)

    def reset_pab_state(self):
        self._stack[0].reset_pab_state()

    def _pos_2d(self, h, w):
        """diffusers PatchEmbed's 2-D sin-cos table for an h x w patch grid (square: h == w)."""
        base = self.config.sample_size // self.patch_size
        s = max(self.config.sample_size // 64, 1)
        return pos_embed_2d(self.inner_dim, (h, w), (base, base), (s, s))

    @torch.no_grad()
    def forward(self, hidden_states, timestep=None, all_timesteps=None, encoder_hidden_states=None, added_cond_kwargs=None,
                class_labels=None, cross_attention_kwargs=None, attention_mask=None, encoder_attention_mask=None,
                use_image_num: int = 0, enable_temporal_attentions: bool = True, return_dict: bool = True, ts_int=None):
        """hidden_states [B, C, F, H, W] latents, timestep [B], encoder_hidden_states [B, L, 4096] (reference :1144-1466)."""
        kernels.require_cuda(hidden_states, "LatteT2V")
        if attention_mask is not None or encoder_attention_mask is not None or use_image_num or not enable_temporal_attentions:
            raise NotImplementedError("masks / joint image training / spatial-only mode are outside the inference path "
                                      "(the reference pipeline never passes them: pipeline_latte.py:854-862)")
        K = kernels
        dt = self.proj_out.weight.dtype
        pm = self.parallel_manager
        cpar = pm is not None and pm.cp_size > 1
        sp = pm is not None and pm.sp_size > 1
        if cpar:  # reference :1198-1216: the CFG pair is split across the cp group
            hidden_states, timestep, encoder_hidden_states = (
                comm.split_sequence(v, pm.cp_group, dim=0) for v in (hidden_states, timestep, encoder_hidden_states))
        B, _, Fr, H, W = hidden_states.shape
        p, C = self.patch_size, self.inner_dim
        h, w = H // p, W // p
        S = h * w
        pos = self.pos_table if S == self.pos_table.shape[1] else self._pos_2d(h, h)[None].to(hidden_states.device)
        x = patch_embed_frames(self.pos_embed, hidden_states, pos, p, dt)  # PatchEmbed (:1245)
        embedded, t6, enc = ada_norm_single(self.adaln_single, self.caption_projection, timestep, encoder_hidden_states, dt)
        if pab_mgr.enable_pab() and ts_int is None:
            ts_int = int(timestep[0])
        if all_timesteps is not None and torch.is_tensor(all_timesteps):
            all_timesteps = all_timesteps.tolist()
        tpe = self.temp_pos_embed[:, :Fr] if Fr > 1 else None
        Fg = Fr
        if sp:  # reference :1300-1308: frames are split (zero-padded to a multiple of sp), the text stays whole
            comm.set_pad("temporal", Fr, pm.sp_group)
            comm.set_pad("spatial", S, pm.sp_group)
            x = comm.split_sequence(x, pm.sp_group, dim=1, pad=comm.get_pad("temporal"))
            if tpe is not None:
                tpe = comm.split_sequence(tpe, pm.sp_group, dim=1, pad=comm.get_pad("temporal"))
            Fr = x.shape[1]
        x = self._stack[0](x, enc, t6, tpe, ts_int=ts_int, all_timesteps=all_timesteps, sp_group=pm.sp_group if sp else None)
        # output head (:1436-1443)
        y = ada_norm_single_out(self.scale_shift_table, embedded, x.view(B, Fr * S, C), B, Fr, S, self.eps)
        y = K.gemm_bias_act(y, self.proj_out.weight, self.proj_out.bias)  # [B, F*S, p*p*Cout]
        if sp:  # the head is row-wise: run on the local frames, gather its 36x narrower output (reference gathers first, :1428-1429)
            y = comm.gather_sequence(y.view(B, Fr, S, -1), pm.sp_group, dim=1, pad=comm.get_pad("temporal"))
            Fr = Fg
        Co = self.out_channels
        y = y.reshape(B * Fr, h, w, p, p, Co)
        y = torch.einsum("nhwpqc->nchpwq", y).reshape(B * Fr, Co, h * p, w * p)
        out = y.reshape(B, Fr, Co, h * p, w * p).permute(0, 2, 1, 3, 4).contiguous()
        if cpar:  # reference :1459-1461
            out = comm.gather_sequence(out, pm.cp_group, dim=0)
        return (out,) if not return_dict else type("Out", (), {"sample": out})()
