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

State-dict compatible with the reference / HF ``LanguageBind/Open-Sora-Plan-v1.2.0`` transformers (``downsampler=None``:
the released 29x480p / 93x480p ... "ROPE-L/122" models) and with checkpoints trained with a conv down-sampler
(``downsampler="k333_s222"``-style: 3-D, or ``"k33_s22"``-style: 2-D, one latent frame only).  Pinned against the reference
file executed unmodified (tests/test_oracle_vs_reference.py::test_osp_v120_*, tests/test_osp_v120_downsampler_cpu.py;
diffusers leaves = the reference's vendored copies).

Down-sampler variants (reference ``Attention`` :653-682, ``DownSampler3d`` / ``DownSampler2d`` :735-834, ``FeedForward_Conv2d``
:1033-1088 chosen at :1273-1288, ``OverlapPatchEmbed3D`` / ``2D`` :372-640): ``vsb_dwconv_shuffle`` runs the depth-wise conv +
shortcut on the modulated tokens and stores them regrouped into dt*dh*dw interleaved sub-grids; self-attention (RoPE3D on
the down-sampled grid) runs inside each sub-grid; ``vsb_gate_residual_unshuffle`` reads the attention output through the
inverse regrouping, so no permutation pass runs, and PAB keeps the regrouped output (replayed through the same kernel).
The feed-forward is project_in with the erf-GELU epilogue, ``vsb_dwconv_ffn`` (h + dw5x5 + dw3x3 + dw1x1 per frame) and
project_out.  The reference's own failures are raised as errors: a latent grid that the down factors do not divide
(ValueError) and the 2-D variant on more than one latent frame (its ``reverse`` folds the frames into the batch).
Sequence parallelism reshapes a token shard as a whole grid in the reference, so it is not offered with a down-sampler.
"""
import re

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


def parse_downsampler(spec):
    """The reference's reading of ``downsampler`` (:655-659): "k<kernel digits>_s<down factor digits>", 2 digits = 2-D
    (per frame), 3 = 3-D.  Returns (kernel, factors) as tuples, or None for no down-sampler."""
    if not spec:
        return None
    k, s = re.search(r"k(\d{2,3})", spec), re.search(r"s(\d{2,3})", spec)
    if k is None or s is None or len(k.group(1)) != len(s.group(1)):
        raise ValueError(f"downsampler {spec!r}: expected k<2 or 3 digits>_s<as many digits>, e.g. 'k333_s222'")
    ks, ds = tuple(int(i) for i in k.group(1)), tuple(int(i) for i in s.group(1))
    kt_ok = len(ks) == 2 or ks[0] in (1, 3)
    if not kt_ok or any(n not in (3, 5) for n in ks[-2:]):
        raise NotImplementedError(f"downsampler {spec!r}: the depth-wise kernel is built for kt in (1, 3) and kh, kw in (3, 5)")
    if 0 in ds:
        raise ValueError(f"downsampler {spec!r}: zero down factor")
    return ks, ds


def _tap_major(cache, key, convs):
    """Depth-wise conv weights [C, 1, *k] as one tap-major [sum of taps, C] copy and the biases as [len(convs), C], kept in
    ``cache`` and rebuilt when a parameter changes (as ``fused_linear``)."""
    ver = tuple((p.data_ptr(), p._version, p.dtype) for m in convs for p in (m.weight, m.bias))
    hit = cache.get(key)
    if hit is None or hit[0] != ver:
        w = torch.cat([m.weight.reshape(m.weight.shape[0], -1).t() for m in convs], 0).contiguous()
        hit = cache[key] = (ver, w, torch.stack([m.bias for m in convs], 0).contiguous())
    return hit[1], hit[2]


class _DownSampler(nn.Module):
    """Parameter holder of DownSampler3d / DownSampler2d (:735-834): a depth-wise conv, "same" padding."""

    def __init__(self, dim, ks):
        super().__init__()
        conv = nn.Conv3d if len(ks) == 3 else nn.Conv2d
        self.layer = conv(dim, dim, kernel_size=ks, stride=1, padding=[(k - 1) // 2 for k in ks], groups=dim)


class _FFConv(nn.Module):
    """Parameter holder of FeedForward_Conv2d (:1033-1088): project_in (C -> 2C), depth-wise 5x5 / 3x3 / 1x1, project_out."""

    def __init__(self, dim):
        super().__init__()
        self.project_in = nn.Linear(dim, 2 * dim)
        self.dwconv = nn.ModuleList([nn.Conv2d(2 * dim, 2 * dim, kernel_size=k, stride=1, padding=k // 2, groups=2 * dim)
                                     for k in (5, 3, 1)])
        self.project_out = nn.Linear(2 * dim, dim)


class OSPBlock(nn.Module):
    def __init__(self, dim, cross_dim, bias=True, ds=None):
        super().__init__()
        self.attn1 = _Attn(dim)
        if ds is not None:
            self.attn1.downsampler = _DownSampler(dim, ds[0])
        self.attn2 = _Attn(dim, cross_dim)
        self.ff = _FF(dim) if ds is None else _FFConv(dim)
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
        self.ds = parse_downsampler(downsampler)
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
                                           hidden_size=dim, cross_attention_dim=cross_attention_dim, downsampler=downsampler))()
        self.inner_dim, self.patch_size, self.out_channels, self.eps, self.use_rope = dim, patch_size, out_channels, norm_eps, use_rope
        st = ((sample_size_t - 1) // 16 + 1) if sample_size_t % 2 == 1 else sample_size_t / 16  # :1574-1583
        self.scale_t = interpolation_scale_t if interpolation_scale_t is not None else st
        self.scale_hw = (interpolation_scale_h if interpolation_scale_h is not None else sample_size[0] / 30,
                         interpolation_scale_w if interpolation_scale_w is not None else sample_size[1] / 40)
        self.pos_embed = PatchEmbed2D(patch_size, in_channels, dim)
        if self.ds is not None and len(self.ds[0]) == 3:  # OverlapPatchEmbed3D (:372-510): Conv3d, kernel = stride = (1, p, p)
            self.pos_embed.proj = nn.Conv3d(in_channels, dim, kernel_size=(1, patch_size, patch_size), stride=(1, patch_size, patch_size))
        self._grid_hw = (sample_size[0] // patch_size, sample_size[1] // patch_size)
        self.num_frames = (sample_size_t - 1) // patch_size_t + 1 if sample_size_t % 2 == 1 else sample_size_t // patch_size_t
        if not use_rope:  # PatchEmbed2D(use_abs_pos=True) :270-283
            self.register_buffer("pos_table", pos_embed_2d(dim, self._grid_hw, self._grid_hw, self.scale_hw)[None], persistent=False)
            tpe = sincos_1d(dim, grid_1d(self.num_frames, self.num_frames, self.scale_t))
            self.register_buffer("temp_pos_embed", tpe.float()[None], persistent=False)
        self.transformer_blocks = nn.ModuleList([OSPBlock(dim, cross_attention_dim, ds=self.ds) for _ in range(num_layers)])
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
        if self.ds is not None and (sp_size or 1) > 1:
            raise NotImplementedError("sequence parallelism with a conv down-sampler (the reference reshapes a token shard as the whole grid)")
        self.parallel_manager = parallel_manager(dp_size, sp_size, enable_cp, self.config.num_attention_heads)

    def reset_pab_state(self):
        for b in self.transformer_blocks:
            b.spatial_count = b.cross_count = 0
            b.spatial_last = b.cross_last = None

    @property
    def _down3(self):
        """(dt, dh, dw) of the down-sampler; the 2-D variant down-samples within each frame (dt = 1)."""
        down = self.ds[1]
        return down if len(down) == 3 else (1, *down)

    def _check_grid(self, pm, T, h, w):
        if pm is not None and pm.sp_size > 1:
            raise NotImplementedError("sequence parallelism with a conv down-sampler (the reference reshapes a token shard as the whole grid)")
        if len(self.ds[1]) == 2 and T > 1:
            raise ValueError(f"downsampler {self.config.downsampler!r} (2-D) runs on one latent frame only, got {T}: the reference's "
                             "DownSampler2d.reverse folds the frames into the batch and fails (open_sora_plan_v120_transformer_3d.py:829-833)")
        dt3, dh, dw = self._down3
        if T % dt3 or h % dh or w % dw:
            raise ValueError(f"downsampler {self.config.downsampler!r}: the latent patch grid {T}x{h}x{w} does not divide by the "
                             f"down factors {dt3}x{dh}x{dw} (the reference's rearrange fails the same way)")

    def _rope_for(self, T, h, w, dtype, device):
        key = (T, h, w, dtype, str(device))
        if key not in self._rope:
            self._rope[key] = rope3d_tables(self.config.attention_head_dim, T, h, w, (self.scale_t, *self.scale_hw), dtype, device)
        return self._rope[key]

    def _run_block(self, blk, x, enc2, mod, B, N, Ng, L, lens, rope, ts_int, sp_group, grid):
        """x [B, N, C] (N = this rank's tokens, Ng = all tokens of a sample); grid = the latent patch grid (T, h, w)."""
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
            nb, n = B, N
            if self.ds is not None:  # conv + shortcut, regrouped into sub-grids of n tokens (:872-874)
                ks, down = self.ds
                wt, bt = _tap_major(blk._fused, "downsampler", [a1.downsampler.layer])
                xm = K.dwconv_shuffle(xm, wt, bt, B, *grid, ks if len(ks) == 3 else (1, *ks), self._down3)
                nb, n = xm.shape[0], xm.shape[1]
            qkv = K.gemm_bias_act(xm.view(nb * n, C), *fused_linear(blk._fused, a1.to_q, a1.to_k, a1.to_v))
            if self.ds is not None:
                if rope is not None:
                    apply_rope_(qkv, rope, H, D, pos_div=1, pos_mod=n)
                o = packed_self_attention(qkv, nb, n, H, D, D**-0.5)
            elif sp_group is None:
                if rope is not None:
                    apply_rope_(qkv, rope, H, D, pos_div=1, pos_mod=N)
                o = packed_self_attention(qkv, B, N, H, D, D**-0.5)
            else:  # tokens for heads (:907-911): every token, H / sp heads; RoPE on the full sequence; back (:937-940)
                o = ulysses_attention(qkv.view(B, N, 3, H, D), 0, Ng, sp_group, D**-0.5, rope=rope)
            a = K.gemm_bias_act(o.view(B * N, C), blk.attn1.to_out[0].weight, blk.attn1.to_out[0].bias)
            if pab_on:
                blk.spatial_last = a
        if self.ds is not None:  # DownSampler.reverse (:959-960) fused into the gate + residual
            K.gate_residual_unshuffle(x, a, mod, 2, B, *grid, self._down3, out=x)
        else:
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
        if self.ds is None:
            hdn = K.gemm_bias_act(xm.view(B * N, C), blk.ff.net[0].proj.weight, blk.ff.net[0].proj.bias, act=1)
            y = K.gemm_bias_act(hdn, blk.ff.net[2].weight, blk.ff.net[2].bias)
        else:  # FeedForward_Conv2d (:1079-1088): project_in + erf-GELU, per-frame depth-wise sum, project_out
            ff = blk.ff
            hdn = K.gemm_bias_act(xm.view(B * N, C), ff.project_in.weight, ff.project_in.bias, act=2)
            wt, bt = _tap_major(blk._fused, "ff.dwconv", list(ff.dwconv))
            T, h, w = grid
            hdn = K.dwconv_ffn(hdn.view(B * T, h, w, 2 * C), wt, bt, B * T, h, w)
            y = K.gemm_bias_act(hdn.view(B * N, 2 * C), ff.project_out.weight, ff.project_out.bias)
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
        if self.ds is not None:
            self._check_grid(pm, Fr, h, w)
        if isinstance(self.pos_embed.proj, nn.Conv3d):  # OverlapPatchEmbed3D: Conv3d on [B, Cin, F, H, W] (:438-442)
            x = self.pos_embed.proj(hidden_states.to(dt)).permute(0, 2, 3, 4, 1).reshape(B * Fr, S, C)
        else:
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
        if self.ds is None:
            rope = self._rope_for(Fr, h, w, dt, hidden_states.device) if self.use_rope else None
        else:  # RoPE3D on the down-sampled grid (:874, :921-925; the 2-D down-sampler sets t = 1)
            dt3, dh, dw = self._down3
            rope = self._rope_for(Fr // dt3, h // dh, w // dw, dt, hidden_states.device) if self.use_rope else None
        Ng = Fr * S
        if sp_group is not None:  # reference :1861-1866 (no padding: the token count must divide)
            x = comm.split_sequence(x, sp_group, dim=1).contiguous()
        N = x.shape[1]
        for blk in self.transformer_blocks:
            mod = K.modulation_table(blk.scale_shift_table, t6, None)
            self._run_block(blk, x, enc2, mod, B, N, Ng, L, lens, rope, ts_int, sp_group, (Fr, h, w))
        y = ada_norm_single_out(self.scale_shift_table, embedded, x, B, 1, N, 1e-6)
        y = K.gemm_bias_act(y.view(B * N, C), self.proj_out.weight, self.proj_out.bias).view(B, N, -1)
        if sp_group is not None:  # the head is row-wise: gather its narrow output (the reference gathers the C-wide rows, :1944-1948)
            y = comm.gather_sequence(y, sp_group, dim=1)
        Co = self.out_channels
        y = y.reshape(B, Fr, h, w, 1, p, p, Co)
        out = torch.einsum("nthwopqc->nctohpwq", y).reshape(B, Co, Fr, h * p, w * p)
        return (out,) if not return_dict else type("Out", (), {"sample": out})()
