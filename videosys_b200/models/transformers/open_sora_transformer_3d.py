"""STDiT3 (OpenSora v1.2) denoiser whose block forward runs on the vsb200 sm_90a kernels.

Drop-in for videosys/models/transformers/open_sora_transformer_3d.py: ``STDiT3Config`` / ``STDiT3`` keep the
constructor arguments, the ``forward(x, timestep, y, all_timesteps, mask, x_mask, fps, height, width)`` signature,
``enable_parallel`` and the exact ``state_dict`` key set / shapes (SURVEY.md Appendix D), so reference checkpoints
load with ``load_state_dict``.  What differs is *how* a step executes (DESIGN.md section 3):

  * every Linear is ``vsb_gemm_bias_act`` (wgmma, bias / tanh-GELU fused in the epilogue);
  * LayerNorm + AdaLN modulate + the t/t0 frame select is ONE pass (``vsb_ln_modulate``), gate + select +
    residual (+ PAB cache write) is ONE pass (``vsb_gate_residual``);
  * spatial / cross attention run ``vsb_attn_flash`` straight on the packed qkv / kv buffers (strided TMA views);
    temporal attention runs ``vsb_attn_short`` on the token-major tensor -- no ``rearrange`` copies anywhere;
  * the PAB gate is evaluated once per block from a HOST integer timestep (one D2H sync per step instead of
    up to three per block: reference :188,190,232), cached tensors are replayed with one ``vsb_residual_add``;
  * the DSP dimension switch is a peer-store kernel (``DspP2P``) with NCCL ``all_to_all_single`` as fallback.

The embedders / final layer (< 2 % of the step, SURVEY.md section 8 row a14) stay as torch ops.
There is no CPU execution path: ``forward`` raises on CPU tensors.
"""
import math
import os
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import kernels
from ...core.distributed import comm
from ...core.distributed.parallel_mgr import ParallelManager
from ...core.pab import pab_mgr
from ._attention import cross_attention, packed_self_attention, temporal_attention
from ._common import parallel_manager, timestep_sinusoid


class STDiT3Config:
    model_type = "STDiT3"

    def __init__(
        self,
        input_size=(None, None, None),
        input_sq_size=512,
        in_channels=4,
        patch_size=(1, 2, 2),
        hidden_size=1152,
        depth=28,
        num_heads=16,
        mlp_ratio=4.0,
        class_dropout_prob=0.1,
        pred_sigma=True,
        drop_path=0.0,
        caption_channels=4096,
        model_max_length=300,
        qk_norm=True,
        enable_flash_attn=False,
        only_train_temporal=False,
        freeze_y_embedder=False,
        skip_y_embedder=False,
        **kwargs,
    ):
        args = dict(locals())
        args.pop("self"), args.pop("kwargs")
        for k, v in args.items():
            setattr(self, k, v)
        for k, v in kwargs.items():
            setattr(self, k, v)


# ---- parameter holders (names/shapes = the reference modules; no forward logic lives here) -------------------
class _NormWeight(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))


class _SelfAttnParams(nn.Module):
    def __init__(self, dim, qk_norm, head_dim):
        super().__init__()
        self.qkv = nn.Linear(dim, dim * 3, bias=True)
        self.q_norm = _NormWeight(head_dim) if qk_norm else nn.Identity()
        self.k_norm = _NormWeight(head_dim) if qk_norm else nn.Identity()
        self.proj = nn.Linear(dim, dim)


class _CrossAttnParams(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.q_linear = nn.Linear(dim, dim)
        self.kv_linear = nn.Linear(dim, dim * 2)
        self.proj = nn.Linear(dim, dim)


class _MlpParams(nn.Module):
    def __init__(self, fin, hidden, fout=None):
        super().__init__()
        self.fc1 = nn.Linear(fin, hidden)
        self.fc2 = nn.Linear(hidden, fout or fin)


class STDiT3Block(nn.Module):
    """Parameters + PAB state of one block (reference :99-150); the forward lives in STDiT3._run_block."""

    def __init__(self, hidden_size, num_heads, mlp_ratio=4.0, qk_norm=False, temporal=False, block_idx=None):
        super().__init__()
        self.temporal = temporal
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.attn = _SelfAttnParams(hidden_size, qk_norm, hidden_size // num_heads)
        self.cross_attn = _CrossAttnParams(hidden_size)
        self.mlp = _MlpParams(hidden_size, int(hidden_size * mlp_ratio))
        self.scale_shift_table = nn.Parameter(torch.randn(6, hidden_size) / hidden_size**0.5)
        self.parallel_manager: Optional[ParallelManager] = None
        self.block_idx = block_idx
        self.reset_pab()

    def reset_pab(self, drop_caches: bool = False):
        """Counters back to zero.  The cache BUFFERS are kept (a count of 0 recomputes and rewrites a cache before any
        step can replay it): captured step graphs hold their addresses, and re-allocating 37 GB of caches per video is
        pointless.  drop_caches=True frees them (shape change, memory pressure)."""
        self.attn_count = 0
        self.cross_count = 0
        if drop_caches or not hasattr(self, "last_attn"):
            self.last_attn = None
            self.last_cross = None


class _Embed2(nn.Module):
    """Linear -> SiLU -> Linear on a 256-wide sinusoid (TimestepEmbedder / SizeEmbedder parameters)."""

    def __init__(self, hidden):
        super().__init__()
        self.mlp = nn.Sequential(nn.Linear(256, hidden), nn.SiLU(), nn.Linear(hidden, hidden))


class _PatchEmbed(nn.Module):
    def __init__(self, patch, cin, hidden):
        super().__init__()
        self.proj = nn.Conv3d(cin, hidden, kernel_size=patch, stride=patch)


class _Caption(nn.Module):
    def __init__(self, cin, hidden, tokens):
        super().__init__()
        self.y_proj = _MlpParams(cin, hidden, hidden)
        self.register_buffer("y_embedding", torch.randn(tokens, cin) / cin**0.5)


class _Final(nn.Module):
    def __init__(self, hidden, out_features):
        super().__init__()
        self.linear = nn.Linear(hidden, out_features)
        self.scale_shift_table = nn.Parameter(torch.randn(2, hidden) / hidden**0.5)


class _Rope(nn.Module):
    def __init__(self, dim, theta=10000.0):
        super().__init__()
        self.freqs = nn.Parameter(1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].float() / dim)), requires_grad=False)


class STDiT3(nn.Module):
    config_class = STDiT3Config
    _fuse_dsp = True  # the P2P switch is always fused into its kernels; bench.py's dsp_parity record reads it as a label

    def __init__(self, config: STDiT3Config):
        super().__init__()
        self.config = config
        C = config.hidden_size
        self.pred_sigma = config.pred_sigma
        self.in_channels = config.in_channels
        self.out_channels = config.in_channels * 2 if config.pred_sigma else config.in_channels
        self.depth, self.hidden_size, self.num_heads = config.depth, C, config.num_heads
        self.mlp_ratio = config.mlp_ratio
        self.patch_size = tuple(config.patch_size)
        self.input_sq_size = config.input_sq_size

        self.rope = _Rope(C // config.num_heads)
        self.x_embedder = _PatchEmbed(self.patch_size, config.in_channels, C)
        self.t_embedder = _Embed2(C)
        self.fps_embedder = _Embed2(C)
        self.t_block = nn.Sequential(nn.SiLU(), nn.Linear(C, 6 * C, bias=True))
        self.y_embedder = _Caption(config.caption_channels, C, config.model_max_length)
        mk = lambda temporal: nn.ModuleList(  # noqa: E731
            [STDiT3Block(C, config.num_heads, config.mlp_ratio, config.qk_norm, temporal, i) for i in range(config.depth)]
        )
        self.spatial_blocks = mk(False)
        self.temporal_blocks = mk(True)
        self.final_layer = _Final(C, int(math.prod(self.patch_size)) * self.out_channels)
        self.initialize_weights()
        self.parallel_manager: Optional[ParallelManager] = None
        self._dsp: Optional[comm.DspP2P] = None
        self._pos_cache = {}
        self._rope_cache = {}
        self._text_cache = None  # per (y, mask): caption MLP output, key layout, per-block kv_linear outputs
        self._hw_cache = None
        self._final_pad = None
        self._fp8 = False

    # ------------------------------------------------------------------------------------------------------
    def initialize_weights(self):
        """Same scheme as the reference (:491-511): xavier-uniform Linears, zero biases, fps_embedder tail and the
        temporal blocks' output projections zero."""
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
        nn.init.normal_(self.fps_embedder.mlp[0].weight, std=0.02)
        nn.init.zeros_(self.fps_embedder.mlp[2].weight)
        for blk in self.temporal_blocks:
            nn.init.zeros_(blk.attn.proj.weight)
            nn.init.zeros_(blk.cross_attn.proj.weight)
            nn.init.zeros_(blk.mlp.fc2.weight)

    @classmethod
    def from_pretrained(cls, path, subfolder: str = "", **config_overrides):
        """STDiT3.from_pretrained (reference pipeline_open_sora.py:222-224) for a LOCAL snapshot directory (config.json +
        safetensors / .bin; videosys_b200/utils/checkpoint.py): the reference's parameter names load strictly."""
        from ...utils.checkpoint import build_from_pretrained

        return build_from_pretrained(cls, path, subfolder, config_cls=STDiT3Config, **config_overrides)

    def enable_parallel(self, dp_size=None, sp_size=None, enable_cp=None, parallel_mgr=None):
        self.parallel_manager = parallel_mgr if parallel_mgr is not None else parallel_manager(dp_size, sp_size, enable_cp)
        for blk in [*self.spatial_blocks, *self.temporal_blocks]:
            blk.parallel_manager = self.parallel_manager

    # ---- FP8 Linears (opt-in) ----------------------------------------------------------------------------------------
    # The block Linears that run on the e4m3 GEMM in FP8 mode: the two whose input the modulate kernel quantizes as it
    # writes it.  The other four need a quantization pass of their own, and with it they lose to the bf16 kernel at
    # 720p (bench_gemm.py, H100 80GB HBM3, 700 W, SM clock 1980 MHz; DESIGN.md section 9): attn.proj 1.51 against
    # 0.76 ms, q_linear 0.66 / 0.57, cross_attn.proj 1.44 / 0.71, fc2 2.39 / 2.33 ms, where qkv (1.35 / 1.65 ms) and
    # fc1 (2.08 / 2.37 ms) win.  kv_linear (once per prompt), the embedders, t_block, the final layer and all attention
    # stay bf16 too.
    FP8_LINEARS = (("attn", "qkv"), ("mlp", "fc1"))

    def _fp8_modules(self):
        for blk in [*self.spatial_blocks, *self.temporal_blocks]:
            for owner, name in self.FP8_LINEARS:
                yield getattr(getattr(blk, owner), name)

    @staticmethod
    def _fp8_refresh(lin: nn.Linear):
        """(Re)quantizes lin's weight into its non-persistent buffers fp8_weight (e4m3 codes, uint8 so that a dtype
        conversion of the module leaves them alone) and fp8_scale (fp32 per output channel) unless they were taken from
        the current parameter: the key follows load_state_dict (the in-place copy bumps _version) and .to() (new
        storage), and a conversion of the scale buffer's dtype is caught by its own check."""
        w = lin.weight
        key = (w.data_ptr(), w._version, w.dtype, w.device)
        sc = lin._buffers.get("fp8_scale")
        if getattr(lin, "_fp8_key", None) == key and sc is not None and sc.dtype == torch.float32 and sc.device == w.device:
            return
        q, scale = kernels.quant_rows_fp8(w.detach())
        lin.register_buffer("fp8_weight", q.view(torch.uint8), persistent=False)
        lin.register_buffer("fp8_scale", scale, persistent=False)
        lin._fp8_key = key

    def set_fp8_linears(self, enabled: bool):
        """FP8 mode: the block Linears FP8_LINEARS of every block run on e4m3 operands -- weights quantized per output
        channel, activations per token row (include/vsb200.h) -- with fp32 accumulation.  Results differ from the
        bf16 path by the quantization.  Disabling restores the bf16 calls exactly.  One GPU only (sp == 1)."""
        pm = self.parallel_manager
        if enabled and pm is not None and pm.sp_size > 1:
            raise NotImplementedError("FP8 Linears under sequence parallelism (the fused DSP modulate would need an fp8 push)")
        self._fp8 = bool(enabled)
        for lin in self._fp8_modules():
            if not enabled:
                for name in ("fp8_weight", "fp8_scale"):
                    lin._buffers.pop(name, None)
                lin._fp8_key = None
            elif lin.weight.is_cuda:  # otherwise at the first forward, once the model is on the GPU
                self._fp8_refresh(lin)
        return self

    def _ln_gemm(self, lin, x, mod, mask_u8, shift_row, scale_row, B, T, S, act=0):
        """lin(ln_modulate(x)) [tanh-GELU]: in FP8 mode the modulate kernel emits the e4m3 rows and their scales, and the
        e4m3 GEMM takes them."""
        if self._fp8:
            qa, sa = kernels.ln_modulate_fp8(x, mod, mask_u8, shift_row, scale_row, B, T, S)
            return kernels.gemm_fp8_bias_act(qa, sa, lin.fp8_weight, lin.fp8_scale, lin.bias, act)
        return kernels.gemm_bias_act(kernels.ln_modulate(x, mod, mask_u8, shift_row, scale_row, B, T, S), lin.weight, lin.bias,
                                     act=act)

    def reset_pab_state(self, drop_caches: bool = False):
        for blk in [*self.spatial_blocks, *self.temporal_blocks]:
            blk.reset_pab(drop_caches)

    def get_dynamic_size(self, x):
        _, _, T, H, W = x.size()
        p = self.patch_size
        return (-(-T // p[0]), -(-H // p[1]), -(-W // p[2]))

    # ---- glue (torch ops; < 2 % of the step) ---------------------------------------------------------------
    def _pos_embed(self, h, w, scale, base_size, dtype, device):
        key = (h, w, float(scale), base_size, dtype, str(device))
        if key not in self._pos_cache:
            half = self.hidden_size // 2
            # the reference keeps inv_freq as a module buffer, so model.to(bf16) rounds it (embeddings.py:236-237)
            inv = (1.0 / (10000 ** (torch.arange(0, half, 2).float() / half))).to(dtype).to(device)
            gh = torch.arange(h, device=device) / scale * (base_size / h)
            gw = torch.arange(w, device=device) / scale * (base_size / w)
            gh, gw = torch.meshgrid(gw, gh, indexing="ij")
            gh, gw = gh.t().reshape(-1), gw.t().reshape(-1)
            sc = lambda v: torch.cat((torch.sin(torch.einsum("i,d->id", v, inv)), torch.cos(torch.einsum("i,d->id", v, inv))), -1)  # noqa: E731
            self._pos_cache[key] = torch.cat([sc(gh), sc(gw)], dim=-1).unsqueeze(0).to(dtype)
        return self._pos_cache[key]

    def _rope_tables(self, n, device):
        key = (n, str(device))
        if key not in self._rope_cache:
            f = self.rope.freqs.float()
            ang = torch.einsum("i,j->ij", torch.arange(n, dtype=torch.float32, device=device), f.to(device))
            ang = ang.repeat_interleave(2, dim=-1)
            self._rope_cache[key] = (ang.cos().contiguous(), ang.sin().contiguous())
        return self._rope_cache[key]

    def _embed(self, emb: _Embed2, v: torch.Tensor, dtype) -> torch.Tensor:
        return emb.mlp(timestep_sinusoid(v).to(dtype))

    def encode_text(self, y, mask=None):
        """Reference STDiT3.encode_text (:526-537): caption MLP, then the mask-compacted [1, sum(lens), C] layout."""
        p = self.y_embedder.y_proj
        y = kernels.gemm_bias_act(kernels.gemm_bias_act(y.contiguous(), p.fc1.weight, p.fc1.bias, act=1), p.fc2.weight,
                                  p.fc2.bias)
        if mask is not None:
            if mask.shape[0] != y.shape[0]:
                mask = mask.repeat(y.shape[0] // mask.shape[0], 1)
            mask = mask.squeeze(1).squeeze(1)
            y = y.squeeze(1).masked_select(mask.unsqueeze(-1) != 0).view(1, -1, self.hidden_size)
            y_lens = mask.sum(dim=1).tolist()
        else:
            y_lens = [y.shape[2]] * y.shape[0]
            y = y.squeeze(1).view(1, -1, self.hidden_size)
        return y, y_lens

    def _text_state(self, y, mask, B, dtype):
        """Timestep-independent text side of the step, computed once per (y, mask) and reused by every denoising step:
        the caption MLP (the reference recomputes it every step, :590), the key layout of the cross-attention and each
        block's kv_linear output.  Returns a dict with y_tok [B*Lv, C], Lv, kv_lens (None = all keys), kv cache.

        Key addressing follows the reference's two implementations:
          * enable_flash_attn=False (default; torch_impl, attentions.py:259-270): the compacted tokens are VIEWED as
            [B, sum(lens)/B] and sample i attends the first min(len_i, sum/B) rows of its slice -- also when the lengths
            differ (the view then crosses sample boundaries; kept bit-for-bit, it is what the reference computes);
          * enable_flash_attn=True (flash_attn_varlen_func with cu_seqlens = cumsum(lens), :240-257): sample i attends
            exactly its own len_i tokens -- here the padded [B, L] layout with per-sample key counts.
        """
        st = self._text_cache
        key = (y._version, None if mask is None or not torch.is_tensor(mask) else mask._version, B, dtype)
        if st is not None and st["y"] is y and st["mask"] is mask and st["key"] == key:
            return st
        y_in = y  # the cache is keyed on the CALLER's tensor (a dtype conversion would make a new object every step)
        y = y if y.dtype == dtype else y.to(dtype)
        C = self.hidden_size
        if self.config.skip_y_embedder:
            y_lens = mask.long().tolist() if isinstance(mask, torch.Tensor) else list(mask)
            y_tok = y.reshape(-1, C).contiguous()
            Lv = y_tok.shape[0] // B
            kv_lens = [min(int(m), Lv) for m in y_lens]
        elif getattr(self.config, "enable_flash_attn", False) and mask is not None:
            p = self.y_embedder.y_proj
            ye = kernels.gemm_bias_act(kernels.gemm_bias_act(y.contiguous(), p.fc1.weight, p.fc1.bias, act=1),
                                       p.fc2.weight, p.fc2.bias).squeeze(1)  # [B, L, C]
            m = mask
            if m.shape[0] != ye.shape[0]:
                m = m.repeat(ye.shape[0] // m.shape[0], 1)
            m = m.reshape(ye.shape[0], -1) != 0
            order = torch.argsort((~m).to(torch.uint8), dim=1, stable=True)  # attendable tokens first, order kept
            y_tok = torch.gather(ye, 1, order[:, :, None].expand(-1, -1, C)).reshape(-1, C).contiguous()
            Lv = ye.shape[1]
            kv_lens = [int(v) for v in m.sum(dim=1).tolist()]
        else:
            y_c, y_lens = self.encode_text(y, mask)
            y_tok = y_c.reshape(-1, C).contiguous()
            Lv = y_tok.shape[0] // B
            kv_lens = [min(int(m), Lv) for m in y_lens]
        if Lv < 1 or min(kv_lens) < 1:
            raise RuntimeError("cross attention needs at least one text token per sample")
        if all(m == Lv for m in kv_lens):
            kv_lens = None
        self._text_cache = dict(y=y_in, mask=mask, key=key, y_tok=y_tok, Lv=Lv, kv_lens=kv_lens, kv={})
        return self._text_cache

    # ---- PAB plan: the per-step skip decisions, taken on the host before anything is launched ------------------------
    def pab_plan(self, ts_int):
        """Evaluates every block's broadcast gate for this step (reference :188-190,232 -> pab_mgr.py:54-91) in
        execution order and ADVANCES the counters.  Returns a tuple of (reuse_attn, reuse_cross) per block, or None when
        PAB is off.  Separating the integer decisions from the launches is what lets a whole step replay as a CUDA
        graph: the plan is the graph's key (core/graph_step.py)."""
        if not pab_mgr.enable_pab():
            return None
        plan = []
        for d in range(self.depth):
            for blk in (self.spatial_blocks[d], self.temporal_blocks[d]):
                gate = pab_mgr.if_broadcast_temporal if blk.temporal else pab_mgr.if_broadcast_spatial
                ra, blk.attn_count = gate(ts_int, blk.attn_count)
                rc, blk.cross_count = pab_mgr.if_broadcast_cross(ts_int, blk.cross_count)
                plan.append((bool(ra), bool(rc)))
        return tuple(plan)

    # ---- one block on the kernels ----------------------------------------------------------------------------
    def _switch(self, x4: torch.Tensor, T: int, S: int, to_spatial_shard: bool) -> torch.Tensor:
        """DSP dimension switch of a [B, t, s, C] tensor (global extents T, S) over all_to_all_single, for process groups
        without CUDA IPC; the P2P path fuses the switch into its kernels (_run_block)."""
        pm = self.parallel_manager
        if to_spatial_shard:
            out = comm.all_to_all_with_pad(x4, pm.sp_group, scatter_dim=2, gather_dim=1,
                                           scatter_pad=comm.get_pad("spatial"), gather_pad=comm.get_pad("temporal"))
        else:
            out = comm.all_to_all_with_pad(x4, pm.sp_group, scatter_dim=1, gather_dim=2,
                                           scatter_pad=comm.get_pad("temporal"), gather_pad=comm.get_pad("spatial"))
        return out.contiguous()  # the narrow() that drops the padding leaves a strided view

    def _run_block(self, blk: STDiT3Block, x, text, t_mlp, t0_mlp, mask_u8, B, T, S, Tg, Sg, plan=(False, False)):
        """x: [B, T*S, C] resident layout (T full, S local); Tg/Sg are the global extents (== T, S when sp == 1).
        text: the dict of _text_state; plan: (reuse_attn, reuse_cross) of this block for this step."""
        K = kernels
        C, H = self.hidden_size, self.num_heads
        D = C // H
        sp = self.parallel_manager.sp_size if self.parallel_manager is not None else 1
        mod = K.modulation_table(blk.scale_shift_table, t_mlp, t0_mlp)
        pab_on = pab_mgr.enable_pab()
        reuse_attn, reuse_cross = plan
        fused_dsp = self._dsp is not None and not blk.temporal and sp > 1

        # ---- self attention ----
        if reuse_attn:
            K.residual_add(x, blk.last_attn, out=x)
        else:
            a = blk.attn
            wq = a.q_norm.weight if hasattr(a.q_norm, "weight") else None
            wk = a.k_norm.weight if hasattr(a.k_norm, "weight") else None
            if wq is None:
                raise RuntimeError("vsb200 STDiT3 kernels implement qk_norm=True (the OpenSora v1.2 configuration)")
            if blk.temporal:
                qkv = self._ln_gemm(a.qkv, x, mod, mask_u8, 0, 1, B, T, S)
                # T < 30: native_attention semantics in one kernel (attentions.py:95-97,111-120); T >= 30: the reference
                # takes F.scaled_dot_product_attention (attentions.py:98-100), same softmax on the flash kernel
                o = temporal_attention(qkv, B, T, S, H, D, D**-0.5, 29, wq, wk, rope=self._rope_tables(T, x.device))
            else:
                Ba = B
                if fused_dsp:
                    # the modulate kernel's stores ARE the S-shard -> T-shard switch (peer stores over NVLink).  It
                    # scatters the B*T (batch, frame) sequences, not the T frames of each sample: spatial attention is
                    # independent per (b, t), and 2*20 = 40 sequences split 8 ways exactly where T = 20 would pad to 24
                    # and leave rank 7 computing only padding (SURVEY.md section 7 "T=20 on 8 GPUs").
                    xm = self._dsp.ln_modulate_push(x, mod, mask_u8, 0, 1, B, T, S, Sg)
                    Ba, Ta, Sa = 1, xm.shape[1], xm.shape[2]
                    xm = xm.reshape(1, Ta * Sa, C)
                elif sp > 1:  # S-sharded -> T-sharded: attention needs every patch of a frame
                    xm = K.ln_modulate(x, mod, mask_u8, 0, 1, B, T, S)
                    xm = self._switch(xm.view(B, T, S, C), Tg, Sg, to_spatial_shard=False)
                    Ta, Sa = xm.shape[1], xm.shape[2]
                    xm = xm.reshape(Ba, Ta * Sa, C)
                else:
                    Ta, Sa = T, S
                if sp > 1:
                    qkv = K.gemm_bias_act(xm, a.qkv.weight, a.qkv.bias)
                else:
                    qkv = self._ln_gemm(a.qkv, x, mod, mask_u8, 0, 1, B, T, S)
                o = packed_self_attention(qkv, Ba * Ta, Sa, H, D, D**-0.5, short_max=29, wq=wq, wk=wk)
            cache = None
            if pab_on:
                if blk.last_attn is None or blk.last_attn.shape != x.shape:
                    blk.last_attn = torch.empty_like(x)
                cache = blk.last_attn
            if not pab_on and (blk.temporal or sp == 1):
                # gate + select + residual in the proj GEMM's epilogue (no PAB cache to fill, no reshard in between)
                K.gemm_bias_residual(o.view(-1, C), a.proj.weight, a.proj.bias, x, mod, mask_u8, 2, B, T, S)
            elif fused_dsp:
                # the branch stays T-sharded in this rank's own window; every rank PULLS the rows of its S-shard in the
                # gate + residual kernel (peer loads over NVLink): the switch back costs no kernel of its own
                K.gemm_bias_act(o.view(-1, C), a.proj.weight, a.proj.bias, out=self._dsp.branch_window(B, T, Sg, C))
                self._dsp.gate_residual_pull(x, mod, mask_u8, 2, B, T, S, Sg, out=x, cache_out=cache)
            else:
                y = K.gemm_bias_act(o.view(-1, C), a.proj.weight, a.proj.bias)
                if not blk.temporal and sp > 1:
                    y = self._switch(y.view(B, Ta, Sa, C), Tg, Sg, to_spatial_shard=True)
                K.gate_residual(x, y.reshape(x.shape), mod, mask_u8, 2, B, T, S, out=x, cache_out=cache)

        # ---- cross attention ----
        if reuse_cross:
            K.residual_add(x, blk.last_cross, out=x)
        else:
            c = blk.cross_attn
            q = K.gemm_bias_act(x, c.q_linear.weight, c.q_linear.bias)
            kv = text["kv"].get(id(blk))
            if kv is None:  # timestep-independent: one kv_linear per block per prompt, not per step
                kv = K.gemm_bias_act(text["y_tok"], c.kv_linear.weight, c.kv_linear.bias)
                text["kv"][id(blk)] = kv
            o = cross_attention(q, kv.view(-1, 2, C), B, T * S, text["Lv"], H, D, D**-0.5, kv_lens=text["kv_lens"])
            if not pab_on:
                K.gemm_bias_residual(o.view(-1, C), c.proj.weight, c.proj.bias, x)  # x += proj(o) in the epilogue
            else:  # PAB: the branch is cached for the steps that reuse it
                out = blk.last_cross if (blk.last_cross is not None and blk.last_cross.shape == x.shape) else None
                blk.last_cross = K.gemm_bias_act(o, c.proj.weight, c.proj.bias, out=out)
                K.residual_add(x, blk.last_cross.view(x.shape), out=x)

        # ---- MLP ----
        h = self._ln_gemm(blk.mlp.fc1, x, mod, mask_u8, 3, 4, B, T, S, act=1)
        K.gemm_bias_residual(h.view(-1, h.shape[-1]), blk.mlp.fc2.weight, blk.mlp.fc2.bias, x, mod, mask_u8, 5, B, T, S)
        return x

    # ---- STDiT3.forward --------------------------------------------------------------------------------------
    def _resolution_sq(self, height, width) -> float:
        """sqrt(height * width) of the first sample as a host float (reference :574: a .item() sync per forward);
        cached per (height, width) tensor pair -- the pipelines pass the same two tensors at every step."""
        c = self._hw_cache
        if c is not None and c[0] is height and c[1] is width and c[2] == (height._version, width._version):
            return c[3]
        v = (height[0].item() * width[0].item()) ** 0.5
        self._hw_cache = (height, width, (height._version, width._version), v)
        return v

    @torch.no_grad()
    def forward(self, x, timestep, y, all_timesteps=None, mask=None, x_mask=None, fps=None, height=None, width=None,
                **kwargs):
        kernels.require_cuda(x, "STDiT3")
        dtype = self.x_embedder.proj.weight.dtype
        if dtype != torch.bfloat16:
            raise RuntimeError("videosys_b200.STDiT3 kernels are bf16: call model.to(torch.bfloat16)")
        pm = self.parallel_manager
        sp = pm.sp_size if pm is not None else 1
        if pm is not None and pm.cp_size > 1:
            raise NotImplementedError("cp (CFG-batch split) is dormant in every reference pipeline (SURVEY 2.2)")
        _, _, Tx, Hx, Wx = x.size()
        T, Hn, Wn = self.get_dynamic_size(x)
        B = x.size(0)
        C = self.hidden_size
        if self._fp8:
            if sp > 1:
                raise NotImplementedError("FP8 Linears under sequence parallelism (the fused DSP modulate would need an fp8 push)")
            for lin in self._fp8_modules():
                self._fp8_refresh(lin)
        if sp > 1 and Tx == 1:
            raise NotImplementedError("image mode (one frame) under sequence parallelism: the reference scatters the "
                                      "batch instead (:292-296); run images on one GPU")
        x = x.to(dtype)
        timestep = timestep.to(dtype)

        # PAB decisions first (host integers); a caller that replays CUDA graphs passes the plan it keyed the graph on
        plan = kwargs.get("pab_plan")
        if plan is None and pab_mgr.enable_pab():
            plan = self.pab_plan(int(timestep[0]))  # the reference's D2H sync, once per step instead of per block

        S = Hn * Wn
        base_size = round(S**0.5)
        pos = self._pos_embed(Hn, Wn, self._resolution_sq(height, width) / self.input_sq_size, base_size, dtype, x.device)

        t = self._embed(self.t_embedder, timestep, dtype)
        f = fps.unsqueeze(1)
        if f.shape[0] != B:
            f = f.repeat(B // f.shape[0], 1)
        fps_e = self._embed(self.fps_embedder, f.reshape(-1), dtype).reshape(B, -1)
        t = t + fps_e
        tb = self.t_block[1]
        t_mlp = kernels.gemm_bias_act(F.silu(t), tb.weight, tb.bias)
        t0 = t0_mlp = None
        mask_u8 = None
        if x_mask is not None:
            t0 = self._embed(self.t_embedder, torch.zeros_like(timestep), dtype) + fps_e
            t0_mlp = kernels.gemm_bias_act(F.silu(t0), tb.weight, tb.bias)
            mask_u8 = x_mask.to(torch.uint8).contiguous()

        text = self._text_state(y, mask, B, dtype)

        # patch embed + position embedding + this rank's patch columns: one kernel (vsb_patch_embed) for temporal patch 1
        # and 16 taps; otherwise the reference's chain (zero pad to the patch grid, strided conv, add, split)
        p = self.patch_size
        Tg, Sg = T, S
        s_pad = 0
        if sp > 1:
            comm.set_pad("temporal", T, pm.sp_group)
            comm.set_pad("spatial", S, pm.sp_group)
            comm.set_pad("batch", B, pm.sp_group)
            s_pad = comm.get_pad("spatial")
        Sl = (S + s_pad) // sp
        h = None
        if p[0] == 1:
            proj = self.x_embedder.proj
            h = kernels.patch_embed(x.contiguous(), proj.weight, proj.bias, pos.reshape(S, C), p[1], p[2],
                                    s0=(pm.sp_rank * Sl if sp > 1 else 0), s_local=Sl)
        if h is None:
            if Wx % p[2]:
                x = F.pad(x, (0, p[2] - Wx % p[2]))
            if Hx % p[1]:
                x = F.pad(x, (0, 0, 0, p[1] - Hx % p[1]))
            if Tx % p[0]:
                x = F.pad(x, (0, 0, 0, 0, 0, p[0] - Tx % p[0]))
            h = self.x_embedder.proj(x).flatten(2).transpose(1, 2)
            h = h.reshape(B, T, S, C) + pos
            if sp > 1:
                h = comm.split_sequence(h, pm.sp_group, dim=2, grad_scale="down", pad=s_pad)
        S = h.shape[2]
        if sp > 1:
            self._ensure_dsp(B, T, S, C, x.device)
        h = h.reshape(B, T * S, C).contiguous()

        depth = kwargs.get("valid_depth", self.depth)
        none = (False, False)
        for d in range(depth):
            ps, pt = (plan[2 * d], plan[2 * d + 1]) if plan is not None else (none, none)
            h = self._run_block(self.spatial_blocks[d], h, text, t_mlp, t0_mlp, mask_u8, B, T, S, Tg, Sg, ps)
            h = self._run_block(self.temporal_blocks[d], h, text, t_mlp, t0_mlp, mask_u8, B, T, S, Tg, Sg, pt)
        if kwargs.get("return_tokens", False):
            return h

        # final layer on the LOCAL S-shard (row-wise ops), then gather its 36x narrower output (reference gathers the
        # C-wide activation first, :615-621: same values, 1/36 of the bytes, and no rank repeats the full-size tail)
        out = self._final_layer(h, t, mask_u8, t0, B, T, S)
        if sp > 1:
            out = comm.gather_sequence(out.reshape(B, T, S, -1), pm.sp_group, dim=2, grad_scale="up",
                                       pad=comm.get_pad("spatial"))
            S = out.shape[2]
            out = out.reshape(B, T * S, -1)
        out = self.unpatchify(out, T, Hn, Wn, Tx, Hx, Wx)
        return out.to(torch.float32)

    def _ensure_dsp(self, B, T, Sl, C, device):
        """Lazily build the P2P windows (largest of the two layouts, padded extents)."""
        if self._dsp is not None or os.environ.get("VSB_DSP_P2P", "1") == "0":
            return
        pm = self.parallel_manager
        w = pm.sp_size
        Tl = -(-(B * T) // w)  # the P2P path scatters the B*T (batch, frame) sequences
        elems = max(B * T * Sl, Tl * Sl * w) * C
        self._dsp = comm.DspP2P(pm.sp_group, elems, device)

    def _final_layer(self, x, t, mask_u8, t0, B, T, S):
        """T2IFinalLayer (reference :75-87), including its quirk: the t0 branch normalises the already
        t-modulated tensor because line :81 rebinds x.  LN + modulate run on vsb_ln_modulate (table rows 0 = shift,
        1 = scale), the 1152 -> 32 projection on the wgmma GEMM."""
        fl = self.final_layer
        C = self.hidden_size
        K = kernels
        tab = fl.scale_shift_table
        tab6 = torch.cat([tab, tab.new_zeros(4, C)], 0)  # the modulate kernel addresses [2, B, 6, C] tables
        z4 = t.new_zeros(B, 4 * C)
        mod = K.modulation_table(tab6, torch.cat([t, t, z4], 1).contiguous(),
                                 None if t0 is None else torch.cat([t0, t0, z4], 1).contiguous())
        out = K.ln_modulate(x, mod[:1].contiguous(), None, 0, 1, B, T, S)  # every frame with the t rows
        if mask_u8 is not None:
            out0 = K.ln_modulate(out, mod[1:].contiguous(), None, 0, 1, B, T, S)
            out = torch.where(mask_u8.bool()[:, :, None, None], out.view(B, T, S, C), out0.view(B, T, S, C)).view(B, T * S, C)
        # 32 output features: run the GEMM's narrowest (64-wide) tile on zero-padded weights, keep the first 32 columns
        w, bias = fl.linear.weight, fl.linear.bias
        n_out = w.shape[0]
        if n_out % 64:
            c = self._final_pad
            if c is None or c[0] != (w._version, bias._version, w.data_ptr()):
                n_pad = -(-n_out // 64) * 64
                wp, bp = w.new_zeros(n_pad, C), bias.new_zeros(n_pad)
                wp[:n_out], bp[:n_out] = w, bias
                c = self._final_pad = ((w._version, bias._version, w.data_ptr()), wp, bp)
            return K.gemm_bias_act(out.contiguous(), c[1], c[2])[..., :n_out]
        return K.gemm_bias_act(out.contiguous(), w, bias)

    def unpatchify(self, x, N_t, N_h, N_w, R_t, R_h, R_w):
        B = x.shape[0]
        Tp, Hp, Wp = self.patch_size
        x = x.reshape(B, N_t, N_h, N_w, Tp, Hp, Wp, self.out_channels)
        x = x.permute(0, 7, 1, 4, 2, 5, 3, 6).reshape(B, self.out_channels, N_t * Tp, N_h * Hp, N_w * Wp)
        return x[:, :, :R_t, :R_h, :R_w]


def STDiT3_XL_2(from_pretrained=None, **kwargs):
    if from_pretrained is not None:
        return STDiT3.from_pretrained(from_pretrained, **kwargs)
    return STDiT3(STDiT3Config(depth=28, hidden_size=1152, patch_size=(1, 2, 2), num_heads=16, **kwargs))
