"""CogVideoX transformer blocks on the vsb200 sm_90a kernels (block level: SURVEY.md section 8 row a15).

``CogVideoXBlockStack`` keeps the reference's state_dict names for ``transformer_blocks.{i}`` (norm1/norm2 =
CogVideoXLayerNormZero: linear + norm; attn1 = diffusers Attention: to_q|to_k|to_v|norm_q|norm_k|to_out.0;
ff.net.0.proj / ff.net.2) and runs CogVideoXBlock.forward (models/transformers/cogvideox_transformer_3d.py:268-312,
attention processor :88-175, sp = 1, no rotary = the 2B model) on the kernels:

  * the two residual streams stay separate ([B, Nv, C] video, [B, Nt, C] text); every LayerNormZero writes its
    modulated output straight into the concatenated [text | video] buffer the joint attention / feed-forward read
    (vsb_ln_modulate_affine on per-sample slices: no torch.cat);
  * to_q / to_k / to_v are one fused GEMM; norm_q / norm_k = vsb_qk_layernorm in place on the packed qkv; the joint
    attention over 226 + 17 550 tokens is vsb_attn_flash (head_dim 64);
  * PAB (spatial gate only, :284-295) caches the un-gated attention output, as the reference does.

Compute dtype: IEEE fp16 (what the reference runs the 2B model in, pipeline_cogvideox.py:138-139; the *_f16 kernel
twins) or bf16 (the 5B model's dtype).  ``CogVideoXTransformer3DModel`` below adds the embedders and the output head
(reference :315-589; the diffusers pieces -- Timesteps, TimestepEmbedding, get_3d_sincos_pos_embed, AdaLayerNorm --
restated from their published semantics, diffusers==0.30.0: parity unpinned for those, SURVEY.md 8c).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import kernels
from ...core.distributed import comm
from ...core.pab import pab_mgr
from ._attention import apply_rope_, packed_self_attention, ulysses_attention
from ._common import fused_linear, parallel_manager, pos_embed_2d, sincos_1d, timestep_sinusoid


class _LayerNormZero(nn.Module):
    def __init__(self, cond_dim, dim, eps=1e-5):
        super().__init__()
        self.linear = nn.Linear(cond_dim, 6 * dim, bias=True)
        self.norm = nn.LayerNorm(dim, eps=eps, elementwise_affine=True)
        self.eps = eps


class _Attn(nn.Module):
    def __init__(self, dim, head_dim, bias=True):
        super().__init__()
        self.to_q = nn.Linear(dim, dim, bias=bias)
        self.to_k = nn.Linear(dim, dim, bias=bias)
        self.to_v = nn.Linear(dim, dim, bias=bias)
        self.norm_q = nn.LayerNorm(head_dim, eps=1e-6)
        self.norm_k = nn.LayerNorm(head_dim, eps=1e-6)
        self.to_out = nn.ModuleList([nn.Linear(dim, dim, bias=True), nn.Identity()])


class _GELUProj(nn.Module):
    def __init__(self, dim, inner):
        super().__init__()
        self.proj = nn.Linear(dim, inner)


class _FF(nn.Module):
    def __init__(self, dim, mult=4):
        super().__init__()
        self.net = nn.ModuleList([_GELUProj(dim, dim * mult), nn.Identity(), nn.Linear(dim * mult, dim), nn.Identity()])


class CogVideoXBlock(nn.Module):
    def __init__(self, dim, heads, head_dim, time_embed_dim, block_idx=0):
        super().__init__()
        self.norm1 = _LayerNormZero(time_embed_dim, dim)
        self.attn1 = _Attn(dim, head_dim, bias=True)
        self.norm2 = _LayerNormZero(time_embed_dim, dim)
        self.ff = _FF(dim)
        self.block_idx = block_idx
        self.attn_count = 0
        self.last_attn = None
        self._fused = {}


class CogVideoXBlockStack(nn.Module):
    def __init__(self, num_attention_heads=30, attention_head_dim=64, num_layers=30, time_embed_dim=512):
        super().__init__()
        self.heads, self.head_dim = num_attention_heads, attention_head_dim
        dim = num_attention_heads * attention_head_dim
        self.dim = dim
        self.transformer_blocks = nn.ModuleList(
            [CogVideoXBlock(dim, num_attention_heads, attention_head_dim, time_embed_dim, i) for i in range(num_layers)]
        )

    def reset_pab_state(self):
        for b in self.transformer_blocks:
            b.attn_count, b.last_attn = 0, None

    def _norm_zero(self, nz: _LayerNormZero, hid, enc, temb, ncat, B, Nv, Nt, C):
        """CogVideoXLayerNormZero for both streams, written into ncat[b] = [text | video]; returns mod [1,B,6,C]
        (rows: shift, scale, gate, enc_shift, enc_scale, enc_gate)."""
        K = kernels
        mod = F.linear(F.silu(temb), nz.linear.weight, nz.linear.bias).view(1, B, 6, C).contiguous()  # tiny (M = B)
        for b in range(B):
            mb = mod[:, b : b + 1]
            K.ln_modulate(enc[b], mb, None, 3, 4, 1, 1, Nt, out=ncat[b, :Nt], eps=nz.eps, gamma=nz.norm.weight, beta=nz.norm.bias)
            K.ln_modulate(hid[b], mb, None, 0, 1, 1, 1, Nv, out=ncat[b, Nt:], eps=nz.eps, gamma=nz.norm.weight, beta=nz.norm.bias)
        return mod

    @torch.no_grad()
    def forward(self, hidden: torch.Tensor, enc: torch.Tensor, temb: torch.Tensor, timestep=None, ts_int=None,
                sp_group=None, n_video: int = None, rope=None):
        """hidden [B, Nv, C], enc [B, Nt, C] (fp16 / bf16, CUDA), temb [B, time_embed_dim]; returns the two streams.
        ts_int: host integer timestep for the PAB gate (else one D2H read of timestep[0], as the reference does).
        sp_group: sequence-parallel group; ``hidden`` is then this rank's chunk of the (zero-padded) video rows and
        ``n_video`` the unpadded global row count.  Everything but the attention core is row-wise and runs on the local
        rows; the joint attention runs on H / sp heads over every row after the head-scatter exchange (reference
        :112-122, :138-143, :162-165), pad rows excluded as keys (:58-62) and zero in the output (:66-72).
        rope (CogVideoX-5b, :146-155): (cos, sin) fp32 tables [text + video rows, head_dim] of ``vsb_qk_rmsnorm_rope``'s RoPE-only
        mode -- identity rows for the text tokens (and pad rows), the 3-D rotary angles for the video tokens; applied to q
        and k after their LayerNorm, on the full sequence."""
        K = kernels
        K.require_cuda(hidden, "CogVideoX blocks", half_only=True)
        B, Nv, C = hidden.shape
        Nt = enc.shape[1]
        N = Nt + Nv
        H, D = self.heads, self.head_dim
        hid = hidden.contiguous().clone()
        en = enc.contiguous().clone()
        ncat = torch.empty(B, N, C, dtype=hid.dtype, device=hid.device)
        pab_on = pab_mgr.enable_pab()
        if ts_int is None:
            ts_int = int(timestep[0]) if (pab_on and timestep is not None) else None
        for blk in self.transformer_blocks:
            mod = self._norm_zero(blk.norm1, hid, en, temb, ncat, B, Nv, Nt, C)
            reuse = False
            if pab_on:
                reuse, blk.attn_count = pab_mgr.if_broadcast_spatial(ts_int, blk.attn_count)
            if reuse:
                a = blk.last_attn
            else:
                at = blk.attn1
                qkv = K.gemm_bias_act(ncat.view(B * N, C), *fused_linear(blk._fused, at.to_q, at.to_k, at.to_v))
                K.qk_layernorm_(qkv, at.norm_q.weight, at.norm_q.bias, at.norm_k.weight, at.norm_k.bias, H, D, eps=1e-6)
                if sp_group is None:
                    if rope is not None:
                        apply_rope_(qkv, rope, H, D, pos_div=1, pos_mod=N)
                    o = packed_self_attention(qkv, B, N, H, D, D**-0.5)
                else:  # every row on H / sp heads; the rope table covers the pad rows with identity
                    o = ulysses_attention(qkv.view(B, N, 3, H, D), Nt, Nt + n_video, sp_group, D**-0.5, rope=rope)
                a = K.gemm_bias_act(o, at.to_out[0].weight, at.to_out[0].bias)  # [B, N, C] = [text | video]
                if pab_on:
                    blk.last_attn = a
            for b in range(B):
                mb = mod[:, b : b + 1]
                K.gate_residual(hid[b], a[b, Nt:], mb, None, 2, 1, 1, Nv, out=hid[b])
                K.gate_residual(en[b], a[b, :Nt], mb, None, 5, 1, 1, Nt, out=en[b])
            mod = self._norm_zero(blk.norm2, hid, en, temb, ncat, B, Nv, Nt, C)
            h = K.gemm_bias_act(ncat.view(B * N, C), blk.ff.net[0].proj.weight, blk.ff.net[0].proj.bias, act=1)
            f = K.gemm_bias_act(h, blk.ff.net[2].weight, blk.ff.net[2].bias).view(B, N, C)
            for b in range(B):
                mb = mod[:, b : b + 1]
                K.gate_residual(hid[b], f[b, Nt:], mb, None, 2, 1, 1, Nv, out=hid[b])
                K.gate_residual(en[b], f[b, :Nt], mb, None, 5, 1, 1, Nt, out=en[b])
        return hid, en


# ---- the whole denoiser (reference CogVideoXTransformer3DModel :315-589), 2B configuration --------------------------------
def get_3d_sincos_pos_embed(embed_dim, spatial_size, temporal_size, spatial_interpolation_scale=1.0,
                            temporal_interpolation_scale=1.0) -> torch.Tensor:
    """diffusers.models.embeddings.get_3d_sincos_pos_embed (0.30.0), call site reference :412-418: a quarter of the
    channels encodes the frame, three quarters the (w-first meshgrid) 2-D position.  Returns [T, H*W, D] float32."""
    assert embed_dim % 4 == 0
    W, H = spatial_size
    d_sp, d_t = 3 * embed_dim // 4, embed_dim // 4
    s = spatial_interpolation_scale
    sp = pos_embed_2d(d_sp, (H, W), (H, W), (s, s))  # [H*W, d_sp]
    tm = sincos_1d(d_t, torch.arange(temporal_size, dtype=torch.float32) / temporal_interpolation_scale)  # [T, d_t]
    out = torch.cat([tm[:, None, :].expand(-1, H * W, -1), sp[None].expand(temporal_size, -1, -1)], dim=-1)
    return out.float()


class _TimestepEmbedding(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.linear_1 = nn.Linear(cin, cout)
        self.linear_2 = nn.Linear(cout, cout)


class _PatchEmbed(nn.Module):
    def __init__(self, patch, cin, dim, text_dim):
        super().__init__()
        self.proj = nn.Conv2d(cin, dim, kernel_size=(patch, patch), stride=patch, bias=True)
        self.text_proj = nn.Linear(text_dim, dim)


class _AdaLayerNorm(nn.Module):
    def __init__(self, cond, dim, eps):
        super().__init__()
        self.linear = nn.Linear(cond, 2 * dim)
        self.norm = nn.LayerNorm(dim, eps, True)


class CogVideoXTransformer3DModel(nn.Module):
    """State-dict compatible with the reference / HF ``THUDM/CogVideoX-2b`` transformer (same module names), forward
    on the vsb200 kernels.  ``enable_parallel`` as the reference: head-scatter sequence parallelism (30 % sp == 0:
    sp in {2, 3, 5, 6, ...}) and CFG parallelism (cp = 2).  ``use_rotary_positional_embeddings`` (CogVideoX-5b: 48 heads x 64,
    42 layers, bf16): no position table is added, ``image_rotary_emb`` rotates q and k of the video tokens."""

    def __init__(self, num_attention_heads=30, attention_head_dim=64, in_channels=16, out_channels=16, flip_sin_to_cos=True,
                 freq_shift=0, time_embed_dim=512, text_embed_dim=4096, num_layers=30, sample_width=90, sample_height=60,
                 sample_frames=49, patch_size=2, temporal_compression_ratio=4, max_text_seq_length=226, norm_eps=1e-5,
                 spatial_interpolation_scale=1.875, temporal_interpolation_scale=1.0,
                 use_rotary_positional_embeddings=False, **unused):
        super().__init__()
        dim = num_attention_heads * attention_head_dim
        self.config = type("Cfg", (), dict(in_channels=in_channels, out_channels=out_channels, patch_size=patch_size,
                                           max_text_seq_length=max_text_seq_length, sample_width=sample_width,
                                           sample_height=sample_height, sample_frames=sample_frames,
                                           use_rotary_positional_embeddings=bool(use_rotary_positional_embeddings),
                                           num_attention_heads=num_attention_heads,
                                           attention_head_dim=attention_head_dim, time_embed_dim=time_embed_dim,
                                           text_embed_dim=text_embed_dim, num_layers=num_layers))()
        self.inner_dim, self.flip, self.freq_shift, self.eps = dim, flip_sin_to_cos, freq_shift, norm_eps
        ph, pw = sample_height // patch_size, sample_width // patch_size
        frames = (sample_frames - 1) // temporal_compression_ratio + 1
        self.num_patches = ph * pw * frames
        self.patch_embed = _PatchEmbed(patch_size, in_channels, dim, text_embed_dim)
        pos = torch.zeros(1, max_text_seq_length + self.num_patches, dim)
        pos[:, max_text_seq_length:] = get_3d_sincos_pos_embed(dim, (pw, ph), frames, spatial_interpolation_scale,
                                                               temporal_interpolation_scale).flatten(0, 1)
        self.register_buffer("pos_embedding", pos, persistent=False)
        self.time_embedding = _TimestepEmbedding(dim, time_embed_dim)
        stack = CogVideoXBlockStack(num_attention_heads, attention_head_dim, num_layers, time_embed_dim)
        self.transformer_blocks = stack.transformer_blocks
        self._stack = [stack]  # not a registered child twice: shares the blocks above
        self.norm_final = nn.LayerNorm(dim, norm_eps, True)
        self.norm_out = _AdaLayerNorm(time_embed_dim, dim, norm_eps)
        self.proj_out = nn.Linear(dim, patch_size * patch_size * out_channels)
        self.parallel_manager = None
        self._rope = None

    def _rope_tables(self, image_rotary_emb, Nt, n_rows, device):
        """(cos, sin) [n_rows, head_dim] fp32: identity for the Nt text rows and for rows past the rotary table (sequence-
        parallel padding), the caller's 3-D rotary angles for the video rows (reference processor :146-155).  Cached on the
        identity of the caller's tensors (the pipeline passes the same pair at every step)."""
        cos, sin = image_rotary_emb
        key = (id(cos), id(sin), cos._version, Nt, n_rows, str(device))
        if self._rope is None or self._rope[0] != key:
            D = self.config.attention_head_dim
            c = torch.ones(n_rows, D, dtype=torch.float32, device=device)
            s_ = torch.zeros(n_rows, D, dtype=torch.float32, device=device)
            n = min(cos.shape[0], n_rows - Nt)
            c[Nt : Nt + n] = cos[:n].to(device=device, dtype=torch.float32)
            s_[Nt : Nt + n] = sin[:n].to(device=device, dtype=torch.float32)
            self._rope = (key, (c.contiguous(), s_.contiguous()))
        return self._rope[1]

    @classmethod
    def from_pretrained(cls, path, subfolder: str = "transformer", **config_overrides):
        """Reference pipeline_cogvideox.py:143-145, for a LOCAL snapshot directory (videosys_b200/utils/checkpoint.py)."""
        from ...utils.checkpoint import build_from_pretrained

        return build_from_pretrained(cls, path, subfolder, **config_overrides)

    def enable_parallel(self, dp_size=None, sp_size=None, enable_cp=None):
        """Reference :462-474."""
        self.parallel_manager = parallel_manager(dp_size, sp_size, enable_cp, self.config.num_attention_heads)

    def reset_pab_state(self):
        self._stack[0].reset_pab_state()

    @torch.no_grad()
    def forward(self, hidden_states, encoder_hidden_states, timestep, timestep_cond=None, image_rotary_emb=None,
                return_dict=True, ts_int=None):
        """hidden_states [B, F, C, H, W] latents, encoder_hidden_states [B, 226, 4096], timestep [B]."""
        K = kernels
        K.require_cuda(hidden_states, "CogVideoX")
        dt = self.proj_out.weight.dtype
        pm = self.parallel_manager
        cp = pm is not None and pm.cp_size > 1
        sp = pm is not None and pm.sp_size > 1
        if cp:  # reference :488-503: the CFG pair is split across the cp group
            hidden_states, encoder_hidden_states, timestep = (
                comm.split_sequence(v, pm.cp_group, dim=0) for v in (hidden_states, encoder_hidden_states, timestep))
        B, Fr, Cin, H, W = hidden_states.shape
        p, C = self.config.patch_size, self.inner_dim
        te = self.time_embedding
        t_emb = timestep_sinusoid(timestep, self.inner_dim, self.flip, self.freq_shift).to(dt)
        emb = K.gemm_bias_act(F.silu(K.gemm_bias_act(t_emb, te.linear_1.weight, te.linear_1.bias)), te.linear_2.weight,
                              te.linear_2.bias)  # [B, 512]
        txt = K.gemm_bias_act(encoder_hidden_states.to(dt).contiguous(), self.patch_embed.text_proj.weight,
                              self.patch_embed.text_proj.bias)  # [B, Nt, C]
        img = self.patch_embed.proj(hidden_states.to(dt).reshape(-1, Cin, H, W))  # conv: cuDNN (glue, once per step)
        img = img.view(B, Fr, C, -1).transpose(2, 3).flatten(1, 2)  # [B, F*h*w, C]
        Nt, Nv = txt.shape[1], img.shape[1]
        if self.config.use_rotary_positional_embeddings:  # reference :519-524: no learned / sin-cos table is added
            enc, hid = txt, img.contiguous()
        else:
            pos = self.pos_embedding[:, : Nt + Nv].to(dt)
            enc = txt + pos[:, :Nt]
            hid = img + pos[:, Nt:]
        if sp:  # reference :531-533: the video rows are split (zero-padded to a multiple of sp), the text rows replicated
            comm.set_pad("pad", Nv, pm.sp_group)
            hid = comm.split_sequence(hid, pm.sp_group, dim=1, pad=comm.get_pad("pad"))
        rope = None
        if image_rotary_emb is not None:
            n_rows = Nt + (hid.shape[1] * pm.sp_size if sp else Nv)  # every row of the gathered sequence, pad rows included
            rope = self._rope_tables(image_rotary_emb, Nt, n_rows, hid.device)
        hid, enc = self._stack[0](hid, enc, emb, timestep, ts_int=ts_int, sp_group=pm.sp_group if sp else None, n_video=Nv,
                                  rope=rope)
        Nv_all, Nv = Nv, hid.shape[1]  # the output head is row-wise: it runs on the local rows, its 30x narrower
        # result is gathered (the reference gathers the C-wide rows first, :563-564: same values)
        # norm_final (plain affine LayerNorm = modulate with shift = scale = 0), then norm_out (AdaLayerNorm, chunk_dim 1:
        # rows shift, scale) and the 1920 -> 64 projection
        zero = torch.zeros(1, B, 6, C, dtype=dt, device=hid.device)
        hid = K.ln_modulate(hid, zero, None, 0, 1, B, 1, Nv, eps=self.eps, gamma=self.norm_final.weight, beta=self.norm_final.bias)
        no = self.norm_out
        ss = K.gemm_bias_act(F.silu(emb), no.linear.weight, no.linear.bias).view(B, 2, C)  # [shift | scale]
        mod = torch.zeros(1, B, 6, C, dtype=dt, device=hid.device)
        mod[0, :, :2] = ss
        hid = K.ln_modulate(hid, mod, None, 0, 1, B, 1, Nv, eps=self.eps, gamma=no.norm.weight, beta=no.norm.bias)
        out = K.gemm_bias_act(hid, self.proj_out.weight, self.proj_out.bias)  # [B, Nv, p*p*Cout]
        if sp:
            out = comm.gather_sequence(out, pm.sp_group, dim=1, pad=comm.get_pad("pad"))
            Nv = Nv_all
        Co = self.config.out_channels
        out = out.reshape(B, Fr, H // p, W // p, Co, p, p).permute(0, 1, 4, 2, 5, 3, 6).flatten(5, 6).flatten(3, 4)
        if cp:  # reference :584-585
            out = comm.gather_sequence(out, pm.cp_group, dim=0)
        return (out,) if not return_dict else type("Out", (), {"sample": out})()
