"""Vchitect-2.0 (VchitectXLTransformerModel) on the vsb200 sm_90a kernels (SURVEY.md section 8 row (f)4).

Reference: models/transformers/vchitect_transformer_3d.py (JointTransformerBlock :50-178, model :237-601) and
models/modules/attentions.py (VchitectAttention :321-638, VchitectAttnProcessor :641-949).  Same module names and
shapes as the reference / HF ``Vchitect/Vchitect-2.0-2B`` transformer (state_dict-compatible).

One MMDiT block keeps two residual streams, video ``[F, S, C]`` and text ``[F, L, C]`` (the text stream is broadcast to
one copy per frame by the first block's AdaLayerNormZero, reference :127-134 with ``temb`` repeated per frame :545-549),
and three attentions over the concatenated ``[video | text]`` tokens of a frame (processor :838-895):

  * temporal (:707-768): every token attends over the F frames at its position, RoPE from ``freqs_cis[:F]``
    (complex multiply on interleaved pairs = the pairing of ``vsb_attn_short`` / ``vsb_qk_rmsnorm_rope``), SDPA rounding,
    no q/k norm: ``vsb_attn_short`` (flags 3; its 64-token instantiation carries the reference's 40-frame example) on the
    token-major tensor, or the RoPE pre-pass + ``vsb_attn_flash`` on strided views beyond 64 frames;
  * cross (:770-803): every token of every frame against the text keys / values of FRAME 0: ``vsb_attn_flash``
    (per-batch key counts);
  * spatial (:663-705): per frame over its S + L tokens: ``vsb_attn_flash``, head_dim 64.

Every Linear is a wgmma GEMM (q|k|v projections of a kind fused into one launch), AdaLayerNormZero /
AdaLayerNormContinuous / norm2 are ``vsb_ln_modulate``, gate + residual is ``vsb_gate_residual``.  What stays torch: the
``[video | text]`` concatenations (strided copies), ``attn * 1.1 + cross`` (:897), the 2-D patch convolution and the
two conditioning MLPs on M = 1 rows.  PAB (temporal, cross, spatial gates in the reference's call order :838-895) caches
exactly the tensors the reference caches.

The diffusers pieces (PatchEmbed with the cropped sin-cos table, CombinedTimestepTextProjEmbeddings, AdaLayerNormZero,
AdaLayerNormContinuous, GELU feed-forward) are restated from their published semantics (diffusers==0.30.0, not
installed).  Pinning: tests/test_oracle_vs_reference.py runs this front end (kernel entries = torch stand-ins) against the
reference's transformer file executed unmodified (test_vchitect_mirror_vs_reference_model, incl. PAB), and the oracle
against the reference's attention class + processor bit for bit.

The reference pipeline calls the transformer with batch 1 (pipeline_vchitect.py:925-941); with a larger batch its
``temb.repeat(F, 1)`` pairs frames with the wrong sample's conditioning, so batch > 1 is rejected here.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import kernels
from ...core.distributed import comm
from ...core.pab import pab_mgr
from ._attention import cross_attention, packed_self_attention, temporal_attention
from ._common import fused_linear, parallel_manager, pos_embed_2d, timestep_sinusoid


# ---- diffusers pieces, restated -----------------------------------------------------------------------------------------

class _PatchEmbed(nn.Module):
    """diffusers PatchEmbed as SD3 / Vchitect use it (layer_norm False, pos_embed_max_size set -> persistent buffer)."""

    def __init__(self, height, width, patch_size, in_channels, embed_dim, pos_embed_max_size):
        super().__init__()
        self.proj = nn.Conv2d(in_channels, embed_dim, kernel_size=(patch_size, patch_size), stride=patch_size, bias=True)
        self.patch_size, self.pos_embed_max_size = patch_size, pos_embed_max_size
        self.base_size = height // patch_size
        m, b = pos_embed_max_size, self.base_size
        pos = pos_embed_2d(embed_dim, (m, m), (b, b), (1.0, 1.0))
        self.register_buffer("pos_embed", pos.unsqueeze(0), persistent=True)

    def cropped_pos_embed(self, height, width):
        h, w, m = height // self.patch_size, width // self.patch_size, self.pos_embed_max_size
        if h > m or w > m:
            raise ValueError(f"latent {height}x{width} exceeds pos_embed_max_size {m}")
        top, left = (m - h) // 2, (m - w) // 2
        return self.pos_embed.reshape(1, m, m, -1)[:, top : top + h, left : left + w, :].reshape(1, h * w, -1)


class _Lin2(nn.Module):
    """TimestepEmbedding / PixArtAlphaTextProjection(act_fn='silu'): linear_1 -> SiLU -> linear_2."""

    def __init__(self, cin, cout):
        super().__init__()
        self.linear_1 = nn.Linear(cin, cout)
        self.linear_2 = nn.Linear(cout, cout)

    def forward(self, x):
        return self.linear_2(F.silu(self.linear_1(x)))


class _TimeTextEmbed(nn.Module):
    """CombinedTimestepTextProjEmbeddings: Timesteps(256, flip_sin_to_cos=True, shift 0) -> TimestepEmbedding, + the pooled
    text projection."""

    def __init__(self, embedding_dim, pooled_projection_dim):
        super().__init__()
        self.timestep_embedder = _Lin2(256, embedding_dim)
        self.text_embedder = _Lin2(pooled_projection_dim, embedding_dim)

    def forward(self, timestep, pooled):
        t = self.timestep_embedder(timestep_sinusoid(timestep).to(pooled.dtype))
        return t + self.text_embedder(pooled)


class _AdaNorm(nn.Module):
    """AdaLayerNormZero (rows = 6: shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp) or
    AdaLayerNormContinuous (rows = 2: scale, shift -- in this order); LayerNorm(eps 1e-6) without affine parameters."""

    def __init__(self, dim, rows):
        super().__init__()
        self.linear = nn.Linear(dim, rows * dim, bias=True)
        self.rows = rows


class _GELUProj(nn.Module):
    def __init__(self, dim, inner):
        super().__init__()
        self.proj = nn.Linear(dim, inner)


class FeedForward(nn.Module):
    """reference :181-234 with activation_fn='gelu-approximate': Linear -> tanh-GELU -> (Dropout) -> Linear."""

    def __init__(self, dim, mult=4):
        super().__init__()
        self.net = nn.ModuleList([_GELUProj(dim, dim * mult), nn.Identity(), nn.Linear(dim * mult, dim)])


class VchitectAttention(nn.Module):
    """Parameter holder with the reference's names (attentions.py:321-523, as JointTransformerBlock builds it: bias on,
    added_kv_proj_dim = dim, no qk norm)."""

    def __init__(self, dim, heads, context_pre_only):
        super().__init__()
        self.heads, self.context_pre_only = heads, context_pre_only
        lin = lambda: nn.Linear(dim, dim, bias=True)  # noqa: E731
        self.to_q, self.to_k, self.to_v = lin(), lin(), lin()
        self.to_q_cross = lin()
        self.to_q_temp, self.to_k_temp, self.to_v_temp = lin(), lin(), lin()
        self.add_k_proj, self.add_v_proj, self.add_q_proj = lin(), lin(), lin()
        self.to_out = nn.ModuleList([lin(), nn.Identity()])
        self.to_out_temporal = lin()
        if not context_pre_only:
            self.to_add_out = lin()
        self.to_add_out_temporal = lin()
        self.to_out_context = lin()
        for m in (self.to_out_temporal, self.to_add_out_temporal, self.to_out_context):  # reference :497-511
            nn.init.zeros_(m.weight)
            nn.init.zeros_(m.bias)
        self.spatial_count = self.temporal_count = self.cross_count = 0
        self.last_spatial = self.last_temporal = self.last_cross = None
        self._fused = {}


class JointTransformerBlock(nn.Module):
    def __init__(self, dim, num_attention_heads, context_pre_only=False):
        super().__init__()
        self.context_pre_only = context_pre_only
        self.norm1 = _AdaNorm(dim, 6)
        self.norm1_context = _AdaNorm(dim, 2 if context_pre_only else 6)
        self.attn = VchitectAttention(dim, num_attention_heads, context_pre_only)
        self.ff = FeedForward(dim)
        if not context_pre_only:
            self.ff_context = FeedForward(dim)


def precompute_freqs_cis(dim: int, end: int, theta: float = 10000.0, rope_scaling_factor: float = 1.0):
    """reference :331-338, returned as (cos, sin) [end, dim] fp32 with every frequency repeated for its (2i, 2i+1) pair."""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: (dim // 2)].float() / dim))
    t = torch.arange(end, dtype=torch.float) / rope_scaling_factor
    ang = torch.outer(t, freqs).float()
    return ang.cos().repeat_interleave(2, dim=1).contiguous(), ang.sin().repeat_interleave(2, dim=1).contiguous()


class VchitectXLTransformerModel(nn.Module):
    def __init__(self, sample_size=128, patch_size=2, in_channels=16, num_layers=18, attention_head_dim=64,
                 num_attention_heads=18, joint_attention_dim=4096, caption_projection_dim=1152, pooled_projection_dim=2048,
                 out_channels=16, pos_embed_max_size=96, rope_scaling_factor=1.0, **unused):
        super().__init__()
        self.out_channels = out_channels if out_channels is not None else in_channels
        self.inner_dim = num_attention_heads * attention_head_dim
        if caption_projection_dim != self.inner_dim:
            raise ValueError("caption_projection_dim must equal heads * head_dim (the blocks add the two streams' projections)")
        self.config = type("Cfg", (), dict(sample_size=sample_size, patch_size=patch_size, in_channels=in_channels,
                                           num_layers=num_layers, attention_head_dim=attention_head_dim,
                                           num_attention_heads=num_attention_heads, joint_attention_dim=joint_attention_dim,
                                           caption_projection_dim=caption_projection_dim,
                                           pooled_projection_dim=pooled_projection_dim, out_channels=self.out_channels,
                                           pos_embed_max_size=pos_embed_max_size, rope_scaling_factor=rope_scaling_factor))()
        C = self.inner_dim
        self.pos_embed = _PatchEmbed(sample_size, sample_size, patch_size, in_channels, C, pos_embed_max_size)
        self.time_text_embed = _TimeTextEmbed(C, pooled_projection_dim)
        self.context_embedder = nn.Linear(joint_attention_dim, caption_projection_dim)
        self.transformer_blocks = nn.ModuleList(
            [JointTransformerBlock(C, num_attention_heads, context_pre_only=(i == num_layers - 1)) for i in range(num_layers)])
        self.norm_out = _AdaNorm(C, 2)
        self.proj_out = nn.Linear(C, patch_size * patch_size * self.out_channels, bias=True)
        self._rope = {}
        self.parallel_manager = None

    # ---- reference surface ----
    @classmethod
    def from_pretrained(cls, path, subfolder: str = "transformer", **config_overrides):
        """reference pipeline_vchitect.py:222-225, for a LOCAL snapshot directory (videosys_b200/utils/checkpoint.py)."""
        from ...utils.checkpoint import build_from_pretrained

        return build_from_pretrained(cls, path, subfolder, **config_overrides)

    def enable_parallel(self, dp_size=None, sp_size=None, enable_cp=None):
        """reference :318-329.  Sequence parallelism shards the FRAMES (:545-549); the temporal attention switches its q / k /
        v to a token shard holding every frame and switches the result back (processor :725-727, :758-759, :929-949; NCCL
        all-to-all).  As in the reference, ``enable_cp`` only takes a factor 2 out of sp_size: the forward never uses the cp
        group (the pipeline runs the two CFG branches one after the other)."""
        self.parallel_manager = parallel_manager(dp_size, sp_size, enable_cp)

    def reset_pab_state(self):
        for b in self.transformer_blocks:
            a = b.attn
            a.spatial_count = a.temporal_count = a.cross_count = 0
            a.last_spatial = a.last_temporal = a.last_cross = None

    def _rope_tables(self, n, device):
        key = (n, str(device))
        if key not in self._rope:
            D = self.config.attention_head_dim
            cos, sin = precompute_freqs_cis(D, n, theta=1e6, rope_scaling_factor=self.config.rope_scaling_factor)
            self._rope[key] = (cos.to(device), sin.to(device))
        return self._rope[key]

    # ---- the attention of one block (VchitectAttnProcessor.__call__) ----
    def _attention(self, a: VchitectAttention, nh, ne, Fr, S, L, ts_int, sp_group=None, Fg=None):
        """nh [Fr, S, C] / ne [Fr, L, C]: the modulated video / text tokens.  Returns (video [Fr*S, C], text [Fr*L, C]).
        sp_group: Fr = this rank's frames, Fg = the video's frames; the temporal attention runs on a token shard with all Fg
        frames (cross attention then uses the text keys of this rank's first frame, cur_frame == 1 is judged on the local
        frame count: the reference's behaviour under sequence parallelism, processor :830-832, :785-786, :906-907)."""
        K = kernels
        C, H = self.inner_dim, a.heads
        D = C // H
        N = S + L
        dev, dt = nh.device, nh.dtype
        scale = D**-0.5
        pab_on = pab_mgr.enable_pab()
        eqkv = K.gemm_bias_act(ne.view(Fr * L, C), *fused_linear(a._fused, a.add_q_proj, a.add_k_proj, a.add_v_proj))
        eqkv = eqkv.view(Fr, L, 3 * C)  # context projections (:823-825)

        # temporal (:838-856)
        reuse = False
        if pab_on:
            reuse, a.temporal_count = pab_mgr.if_broadcast_temporal(ts_int, a.temporal_count)
        if reuse:
            hid_t, enc_t = a.last_temporal
        else:
            w, b = fused_linear(a._fused, a.to_q_temp, a.to_k_temp, a.to_v_temp)
            jt = torch.empty(Fr, N, 3 * C, dtype=dt, device=dev)
            jt[:, :S] = K.gemm_bias_act(nh.view(Fr * S, C), w, b).view(Fr, S, 3 * C)
            jt[:, S:] = eqkv
            Ft, Nt = Fr, N  # frames / tokens the temporal attention sees
            if sp_group is not None:  # frame shard -> token shard (scatter the tokens, gather the frames)
                comm.set_pad("spatial", N, sp_group)
                jt = comm.all_to_all_with_pad(jt.view(1, Fr, N, 3 * C), sp_group, scatter_dim=2, gather_dim=1,
                                              scatter_pad=comm.get_pad("spatial"), gather_pad=comm.get_pad("temporal")).contiguous()
                Ft, Nt = jt.shape[1], jt.shape[2]
                jt = jt.view(Ft, Nt, 3 * C)
            ot = temporal_attention(jt, 1, Ft, Nt, H, D, scale, 64, rope=self._rope_tables(Ft, dev), sdpa=True)
            if sp_group is not None:  # token shard -> frame shard
                ot = comm.all_to_all_with_pad(ot.view(1, Ft, Nt, C), sp_group, scatter_dim=1, gather_dim=2,
                                              scatter_pad=comm.get_pad("temporal"), gather_pad=comm.get_pad("spatial")).contiguous()
            ot = ot.view(Fr, N, C)
            hid_t = K.gemm_bias_act(ot[:, :S].contiguous().view(Fr * S, C), a.to_out_temporal.weight, a.to_out_temporal.bias)
            enc_t = ot[:, S:].contiguous().view(Fr * L, C)
            if pab_on:
                a.last_temporal = (hid_t, enc_t)

        # cross (:858-877): all tokens of all frames against frame 0's text keys / values
        reuse = False
        if pab_on:
            reuse, a.cross_count = pab_mgr.if_broadcast_cross(ts_int, a.cross_count)
        if reuse:
            cross = a.last_cross
        else:
            jc = torch.empty(Fr, N, C, dtype=dt, device=dev)
            jc[:, :S] = K.gemm_bias_act(nh.view(Fr * S, C), a.to_q_cross.weight, a.to_q_cross.bias).view(Fr, S, C)
            jc[:, S:] = eqkv[:, :, :C]
            oc = cross_attention(jc, eqkv[0].view(L, 3, C), 1, Fr * N, L, H, D, scale)
            cross = K.gemm_bias_act(oc.view(Fr * N, C), a.to_out_context.weight, a.to_out_context.bias)
            if pab_on:
                a.last_cross = cross

        # spatial (:879-895)
        reuse = False
        if pab_on:
            reuse, a.spatial_count = pab_mgr.if_broadcast_spatial(ts_int, a.spatial_count)
        if reuse:
            sp_out = a.last_spatial
        else:
            w, b = fused_linear(a._fused, a.to_q, a.to_k, a.to_v)
            js = torch.empty(Fr, N, 3 * C, dtype=dt, device=dev)
            js[:, :S] = K.gemm_bias_act(nh.view(Fr * S, C), w, b).view(Fr, S, 3 * C)
            js[:, S:] = eqkv
            sp_out = packed_self_attention(js, Fr, N, H, D, scale).view(Fr * N, C)
            if pab_on:
                a.last_spatial = sp_out

        mix = (sp_out * 1.1 + cross).view(Fr, N, C)  # :897
        hv = K.gemm_bias_act(mix[:, :S].contiguous().view(Fr * S, C), a.to_out[0].weight, a.to_out[0].bias)
        if Fr == 1:  # :906-907, :914-915
            hid_t = hid_t * 0
        hv = K.residual_add(hv, hid_t.view(Fr * S, C))
        he = mix[:, S:].contiguous().view(Fr * L, C)
        if not a.context_pre_only:
            he = K.gemm_bias_act(he, a.to_add_out.weight, a.to_add_out.bias)
        et = K.gemm_bias_act(enc_t, a.to_add_out_temporal.weight, a.to_add_out_temporal.bias)
        if Fr == 1:
            et = et * 0
        he = K.residual_add(he, et)
        return hv, he

    def _mod(self, nz: _AdaNorm, temb):
        """linear(silu(temb)) laid out as the [1, 1, rows, C] table the modulate / gate kernels read."""
        return kernels.gemm_bias_act(F.silu(temb), nz.linear.weight, nz.linear.bias).view(1, 1, nz.rows, self.inner_dim)

    def _run_block(self, blk: JointTransformerBlock, hid, enc, temb, Fr, S, L, ts_int, sp_group=None, Fg=None):
        """hid [Fr*S, C]; enc [Fr*L, C] (or [L, C] before the first block); returns the two streams."""
        K = kernels
        C = self.inner_dim
        mod = self._mod(blk.norm1, temb)
        nh = K.ln_modulate(hid, mod, None, 0, 1, 1, Fr, S, eps=1e-6)
        if enc.shape[0] == L and Fr > 1:  # first block: one text copy per frame from here on (broadcast in norm1_context)
            enc = enc.view(1, L, C).expand(Fr, L, C).contiguous().view(Fr * L, C)
        if blk.context_pre_only:
            cmod = self._mod(blk.norm1_context, temb)  # rows: scale, shift
            ne = K.ln_modulate(enc, cmod, None, 1, 0, 1, Fr, L, eps=1e-6)
        else:
            cmod = self._mod(blk.norm1_context, temb)
            ne = K.ln_modulate(enc, cmod, None, 0, 1, 1, Fr, L, eps=1e-6)
        hv, he = self._attention(blk.attn, nh.view(Fr, S, C), ne.view(Fr, L, C), Fr, S, L, ts_int, sp_group, Fg)
        hid = K.gate_residual(hid, hv, mod, None, 2, 1, Fr, S)
        nh = K.ln_modulate(hid, mod, None, 3, 4, 1, Fr, S, eps=1e-6)
        f = K.gemm_bias_act(K.gemm_bias_act(nh, blk.ff.net[0].proj.weight, blk.ff.net[0].proj.bias, act=1),
                            blk.ff.net[2].weight, blk.ff.net[2].bias)
        hid = K.gate_residual(hid, f, mod, None, 5, 1, Fr, S)
        if blk.context_pre_only:
            return hid, None
        enc = K.gate_residual(enc, he, cmod, None, 2, 1, Fr, L)
        ne = K.ln_modulate(enc, cmod, None, 3, 4, 1, Fr, L, eps=1e-6)
        f = K.gemm_bias_act(K.gemm_bias_act(ne, blk.ff_context.net[0].proj.weight, blk.ff_context.net[0].proj.bias, act=1),
                            blk.ff_context.net[2].weight, blk.ff_context.net[2].bias)
        enc = K.gate_residual(enc, f, cmod, None, 5, 1, Fr, L)
        return hid, enc

    @torch.no_grad()
    def forward(self, hidden_states, encoder_hidden_states=None, pooled_projections=None, timestep=None,
                joint_attention_kwargs=None, return_dict: bool = True, ts_int=None):
        """hidden_states [1, F, C_in, H, W] latents, encoder_hidden_states [1, L, joint_attention_dim],
        pooled_projections [1, pooled_projection_dim], timestep [1]; returns ``sample`` [F, C_out, H, W] (reference
        :478-601).  ts_int: host integer timestep for the PAB gates (else one D2H read of ``timestep[0]``, as the
        reference does three times per block)."""
        K = kernels
        K.require_cuda(hidden_states, "Vchitect")
        dt = self.proj_out.weight.dtype
        B, Fr, Cin, Hh, Ww = hidden_states.shape
        if B != 1:
            raise ValueError("videosys_b200 Vchitect: one sample per forward (the reference pipeline calls the transformer "
                             "with batch 1; its per-frame conditioning repeat is only consistent for batch 1)")
        p, C = self.config.patch_size, self.inner_dim
        pe = self.pos_embed
        x = pe.proj(hidden_states.to(dt).reshape(Fr, Cin, Hh, Ww))  # conv: cuDNN (glue, once per step)
        x = x.flatten(2).transpose(1, 2)  # [F, S, C]
        hid = (x + pe.cropped_pos_embed(Hh, Ww).to(x.dtype)).to(dt).contiguous()
        S = hid.shape[1]
        temb = self.time_text_embed(timestep, pooled_projections.to(dt))  # [1, C] (M = 1 rows: torch)
        enc = K.gemm_bias_act(encoder_hidden_states.to(dt).contiguous(), self.context_embedder.weight, self.context_embedder.bias)
        L = enc.shape[1]
        pm = self.parallel_manager
        sp_group = pm.sp_group if (pm is not None and pm.sp_size > 1) else None
        Fg = Fr
        if sp_group is not None:  # reference :545-549: this rank's frames (zero frames pad the last rank)
            comm.set_pad("temporal", Fr, sp_group)
            hid = comm.split_sequence(hid.view(1, Fr, S, C), sp_group, dim=1, pad=comm.get_pad("temporal")).contiguous()
            Fr = hid.shape[1]
        hid, enc = hid.view(Fr * S, C), enc.view(L, C)
        if ts_int is None and pab_mgr.enable_pab():
            ts_int = int(timestep[0])
        for blk in self.transformer_blocks:
            hid, enc = self._run_block(blk, hid, enc, temb, Fr, S, L, ts_int, sp_group, Fg)
        omod = self._mod(self.norm_out, temb)  # AdaLayerNormContinuous: rows scale, shift
        hid = K.ln_modulate(hid, omod, None, 1, 0, 1, Fr, S, eps=1e-6)
        out = K.gemm_bias_act(hid, self.proj_out.weight, self.proj_out.bias)  # [F*S, p*p*Cout]
        if sp_group is not None:  # the head is row-wise: gather its narrow output (the reference gathers the C-wide rows, :563-564)
            out = comm.gather_sequence(out.view(1, Fr, S, -1), sp_group, dim=1, pad=comm.get_pad("temporal"))
            Fr = Fg
            out = out.reshape(Fr * S, -1)
        Co, h, w = self.out_channels, Hh // p, Ww // p
        out = out.view(Fr, h, w, p, p, Co).permute(0, 5, 1, 3, 2, 4).reshape(Fr, Co, h * p, w * p)  # nhwpqc -> nchpwq
        return (out,) if not return_dict else type("Out", (), {"sample": out})()
