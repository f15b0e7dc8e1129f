"""TEST INFRASTRUCTURE ONLY -- loads the *unmodified* reference modules for oracle pinning.

Imports VideoSys' OpenSora hot-path modules straight from the reference tree (``VSB_REFERENCE_ROOT``, read-only) by
registering a bare ``videosys`` namespace package (skipping ``videosys/__init__.py:1-12`` which
pulls every pipeline -> diffusers) and stubbing the third-party names that are not installed in
this image (timm ``Mlp``/``DropPath``, colossalai ``ProcessGroupMesh``, diffusers ``Attention``,
``rotary_embedding_torch.RotaryEmbedding``, imageio, omegaconf).  Recipe: SURVEY.md Appendix C.

Only ``tests/`` and ``oracle/gen_golden.py`` may import this file, and only inside the authoring
machine that has the reference tree; elsewhere ``available()`` says it is absent.
"""
import importlib
import os
import sys
import types

import torch
import torch.nn as nn

REF = os.environ.get("VSB_REFERENCE_ROOT", "/root/reference")


def available() -> bool:
    return os.path.isdir(os.path.join(REF, "videosys"))


def _mod(name, **kw):
    m = types.ModuleType(name)
    m.__dict__.update(kw)
    sys.modules[name] = m
    return m


class _Mlp(nn.Module):
    """timm.models.vision_transformer.Mlp semantics: fc2(act(fc1(x))), biases on, dropout 0."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0, **_):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features, out_features)

    def forward(self, x):
        return self.fc2(self.act(self.fc1(x)))


class _RotaryEmbedding(nn.Module):
    """rotary_embedding_torch.RotaryEmbedding(dim) ('lang' freqs, theta 1e4), rotate_queries_or_keys only."""

    def __init__(self, dim, theta=10000):
        super().__init__()
        self.freqs = nn.Parameter(
            1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].float() / dim)), requires_grad=False
        )

    def rotate_queries_or_keys(self, t, seq_dim=-2):
        n = t.shape[seq_dim]
        pos = torch.arange(n, device=t.device, dtype=torch.float32)
        f = torch.einsum("i,j->ij", pos, self.freqs.float()).repeat_interleave(2, dim=-1)
        x1, x2 = t.reshape(*t.shape[:-1], -1, 2).unbind(-1)
        rh = torch.stack((-x2, x1), -1).flatten(-2)
        return (t * f.cos() + rh * f.sin()).type(t.dtype)


_LOADED = {}


def load():
    """Returns a namespace with the reference modules (cached)."""
    if _LOADED:
        return types.SimpleNamespace(**_LOADED)
    if not available():
        raise RuntimeError(f"reference tree not present at {REF}")
    import transformers  # noqa: F401  (must be imported before timm is stubbed)

    pkg = _mod("videosys")
    pkg.__path__ = [REF + "/videosys"]
    _mod("timm")
    _mod("timm.models")
    _mod("timm.models.layers", DropPath=nn.Identity)
    _mod("timm.models.vision_transformer", Mlp=_Mlp)
    _mod("colossalai")
    _mod("colossalai.cluster")
    _mod(
        "colossalai.cluster.process_group_mesh",
        ProcessGroupMesh=type("ProcessGroupMesh", (), {"__init__": lambda s, *a: None}),
    )
    _mod("diffusers")
    _mod("diffusers.models")
    _mod("diffusers.models.attention", Attention=object)
    _mod("diffusers.models.attention_processor", AttnProcessor=object)
    _mod("imageio")
    _mod("omegaconf", DictConfig=dict, ListConfig=list, OmegaConf=object)
    _mod("rotary_embedding_torch", RotaryEmbedding=_RotaryEmbedding)
    _LOADED["stdit3"] = importlib.import_module("videosys.models.transformers.open_sora_transformer_3d")
    _LOADED["attentions"] = importlib.import_module("videosys.models.modules.attentions")
    _LOADED["normalization"] = importlib.import_module("videosys.models.modules.normalization")
    _LOADED["pab_mgr"] = importlib.import_module("videosys.core.pab.pab_mgr")
    _LOADED["comm"] = importlib.import_module("videosys.core.distributed.comm")
    _LOADED["rflow"] = importlib.import_module("videosys.schedulers.scheduling_rflow_open_sora")
    return types.SimpleNamespace(**_LOADED)


class SingleRankPM:
    """Stand-in for ParallelManager on one rank (parallel_mgr.py:14-39)."""

    sp_size = 1
    cp_size = 1
    sp_group = None
    cp_group = None


def build_stdit3(depth=1, hidden_size=1152, num_heads=16, dtype=torch.float32, **kw):
    ref = load()
    M = ref.stdit3
    net = M.STDiT3(M.STDiT3Config(depth=depth, hidden_size=hidden_size, num_heads=num_heads, **kw)).eval().to(dtype)
    net.parallel_manager = SingleRankPM()
    for b in [*net.spatial_blocks, *net.temporal_blocks]:
        b.parallel_manager = SingleRankPM()
    return net


def load_cogvideox_scheduler():
    """The reference's CogVideoXDDIMScheduler class (schedulers/scheduling_ddim_cogvideox.py), imported unmodified with
    the three diffusers base names it needs stubbed (ConfigMixin / register_to_config: keep the constructor kwargs as
    ``self.config``; SchedulerMixin; BaseOutput).  All scheduler arithmetic is the reference's own."""
    import functools
    import inspect

    if not available():
        raise RuntimeError(f"reference tree not present at {REF}")
    if "videosys" not in sys.modules:
        pkg = _mod("videosys")
        pkg.__path__ = [REF + "/videosys"]

    def register_to_config(init):
        @functools.wraps(init)
        def wrapper(self, *a, **kw):
            sig = inspect.signature(init)
            bound = sig.bind(self, *a, **kw)
            bound.apply_defaults()
            self.config = types.SimpleNamespace(**{k: v for k, v in bound.arguments.items() if k != "self"})
            init(self, *a, **kw)

        return wrapper

    class BaseOutput:
        def __init_subclass__(cls, **kw):
            super().__init_subclass__(**kw)

    for name in ("diffusers", "diffusers.schedulers"):
        if name not in sys.modules:
            _mod(name)
    _mod("diffusers.configuration_utils", ConfigMixin=type("ConfigMixin", (), {}), register_to_config=register_to_config)
    _mod("diffusers.schedulers.scheduling_utils", KarrasDiffusionSchedulers=[], SchedulerMixin=type("SchedulerMixin", (), {}))
    _mod("diffusers.utils", BaseOutput=BaseOutput)
    return importlib.import_module("videosys.schedulers.scheduling_ddim_cogvideox").CogVideoXDDIMScheduler


# ---- Open-Sora-Plan v1.1.0: the reference module imported unmodified, diffusers LEAF classes restated --------------------------
class _RefGELU(nn.Module):
    """diffusers.models.activations.GELU(dim_in, dim_out, approximate, bias): Linear then F.gelu."""

    def __init__(self, dim_in, dim_out, approximate="none", bias=True):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out, bias=bias)
        self.approximate = approximate

    def forward(self, x, *a, **k):
        return torch.nn.functional.gelu(self.proj(x), approximate=self.approximate)


class _RefTimesteps(nn.Module):
    """diffusers Timesteps(num_channels, flip_sin_to_cos, downscale_freq_shift): get_timestep_embedding, scale 1."""

    def __init__(self, num_channels, flip_sin_to_cos, downscale_freq_shift):
        super().__init__()
        self.n, self.flip, self.shift = num_channels, flip_sin_to_cos, downscale_freq_shift

    def forward(self, timesteps):
        import math

        half = self.n // 2
        exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32, device=timesteps.device) / (half - self.shift)
        emb = timesteps[:, None].float() * torch.exp(exponent)[None, :]
        emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
        return torch.cat([emb[:, half:], emb[:, :half]], dim=-1) if self.flip else emb


class _RefTimestepEmbedding(nn.Module):
    """diffusers TimestepEmbedding(in_channels, time_embed_dim): linear_1 -> SiLU -> linear_2."""

    def __init__(self, in_channels, time_embed_dim, act_fn="silu", **_):
        super().__init__()
        assert act_fn == "silu"
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)

    def forward(self, sample, condition=None):
        return self.linear_2(self.act(self.linear_1(sample)))


def _register_to_config(init):
    import functools
    import inspect

    @functools.wraps(init)
    def wrapper(self, *a, **kw):
        bound = inspect.signature(init).bind(self, *a, **kw)
        bound.apply_defaults()
        self.__dict__["config"] = types.SimpleNamespace(**{k: v for k, v in bound.arguments.items() if k != "self"})
        init(self, *a, **kw)

    return wrapper


class _ModelMixin(nn.Module):
    @property
    def dtype(self):
        return next(self.parameters()).dtype


def load_osp_v110():
    """The reference's models/transformers/open_sora_plan_v110_transformer_3d.py, imported unmodified.  Everything the file
    defines itself (RoPE1D/2D, PatchEmbed, Attention + AttnProcessor2_0, FeedForward, both block classes, AdaLayerNormSingle,
    CaptionProjection, LatteT2V) runs as written; of the diffusers names it imports only three leaf classes carry arithmetic
    on the inference path and are restated here (GELU, Timesteps, TimestepEmbedding); the rest are placeholders."""
    if "osp_v110" in _LOADED:
        return _LOADED["osp_v110"]
    load()  # videosys namespace + the shared stubs
    ph = lambda name: type(name, (nn.Module,), {})  # noqa: E731  (placeholder class: never instantiated on this path)
    _mod("diffusers.configuration_utils", ConfigMixin=type("ConfigMixin", (), {}), register_to_config=_register_to_config)
    _mod("diffusers.models.activations", GEGLU=ph("GEGLU"), GELU=_RefGELU, ApproximateGELU=ph("ApproximateGELU"))
    names = ["AttnAddedKVProcessor", "AttnAddedKVProcessor2_0", "AttnProcessor", "CustomDiffusionAttnProcessor",
             "CustomDiffusionAttnProcessor2_0", "CustomDiffusionXFormersAttnProcessor", "LoRAAttnAddedKVProcessor",
             "LoRAAttnProcessor", "LoRAAttnProcessor2_0", "LoRAXFormersAttnProcessor", "SlicedAttnAddedKVProcessor",
             "SlicedAttnProcessor", "SpatialNorm", "XFormersAttnAddedKVProcessor", "XFormersAttnProcessor"]
    _mod("diffusers.models.attention_processor", **{n: ph(n) for n in names})
    _mod("diffusers.models.embeddings", SinusoidalPositionalEmbedding=ph("SinusoidalPositionalEmbedding"),
         TimestepEmbedding=_RefTimestepEmbedding, Timesteps=_RefTimesteps)
    _mod("diffusers.models.lora", LoRACompatibleConv=nn.Conv2d, LoRACompatibleLinear=nn.Linear)
    _mod("diffusers.models.modeling_utils", ModelMixin=_ModelMixin)
    _mod("diffusers.models.normalization", AdaLayerNorm=ph("AdaLayerNorm"), AdaLayerNormZero=ph("AdaLayerNormZero"))
    _mod("diffusers.utils", USE_PEFT_BACKEND=True, BaseOutput=type("BaseOutput", (), {}), deprecate=lambda *a, **k: None,
         is_xformers_available=lambda: False)
    _mod("diffusers.utils.torch_utils", maybe_allow_in_graph=lambda cls: cls)
    m = importlib.import_module("videosys.models.transformers.open_sora_plan_v110_transformer_3d")
    _LOADED["osp_v110"] = m
    return m


def build_osp_v110(dtype=torch.float32, **cfg):
    M = load_osp_v110()
    net = M.LatteT2V(**cfg).eval().to(dtype)
    net.parallel_manager = SingleRankPM()
    for mod in net.modules():
        if hasattr(mod, "parallel_manager"):
            mod.parallel_manager = SingleRankPM()
    return net


def load_latte():
    """The reference's models/transformers/latte_transformer_3d.py, imported unmodified.  Its diffusers leaf classes are
    taken from the REFERENCE'S OWN vendored copies in open_sora_plan_v110_transformer_3d.py (same authors, same semantics:
    Attention + AttnProcessor2_0 with RoPE off, PatchEmbed, CombinedTimestepSizeEmbeddings, CaptionProjection,
    get_1d_sincos_pos_embed_from_grid) plus the three restated leaves of load_osp_v110 (GELU, Timesteps, TimestepEmbedding)."""
    if "latte" in _LOADED:
        return _LOADED["latte"]
    O = load_osp_v110()

    class Attention(O.Attention):  # diffusers' constructor signature -> the vendored class (RoPE / KV compression off)
        def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=64, dropout=0.0, bias=False,
                     upcast_attention=False, out_bias=True, **kw):
            super().__init__(query_dim=query_dim, cross_attention_dim=cross_attention_dim, heads=heads, dim_head=dim_head,
                             dropout=dropout, bias=bias, upcast_attention=upcast_attention, out_bias=out_bias,
                             attention_mode="math", use_rope=False, rope_scaling=None, compress_kv_factor=None, **kw)

    class PixArtAlphaTextProjection(O.CaptionProjection):  # the diffusers class has no y_embedding buffer
        def __init__(self, in_features, hidden_size, **kw):
            super().__init__(in_features, hidden_size)
            del self._buffers["y_embedding"]

    ph = lambda name: type(name, (nn.Module,), {})  # noqa: E731
    sys.modules["diffusers.models.attention_processor"].Attention = Attention
    emb = sys.modules["diffusers.models.embeddings"]
    emb.ImagePositionalEmbeddings = ph("ImagePositionalEmbeddings")
    emb.PatchEmbed = O.PatchEmbed
    emb.PixArtAlphaCombinedTimestepSizeEmbeddings = O.CombinedTimestepSizeEmbeddings
    emb.PixArtAlphaTextProjection = PixArtAlphaTextProjection
    emb.get_1d_sincos_pos_embed_from_grid = O.get_1d_sincos_pos_embed_from_grid
    sys.modules["diffusers.models.normalization"].AdaLayerNormContinuous = ph("AdaLayerNormContinuous")
    m = importlib.import_module("videosys.models.transformers.latte_transformer_3d")
    _LOADED["latte"] = m
    return m


def build_latte(dtype=torch.float32, **cfg):
    M = load_latte()
    net = M.LatteT2V(**cfg).eval().to(dtype)
    net.parallel_manager = SingleRankPM()
    for mod in net.modules():
        if hasattr(mod, "parallel_manager"):
            mod.parallel_manager = SingleRankPM()
    return net


def load_cogvideox():
    """The reference's models/transformers/cogvideox_transformer_3d.py (+ its in-tree CogVideoXPatchEmbed,
    CogVideoXLayerNormZero, AdaLayerNorm, CogVideoXAttnProcessor2_0), imported unmodified.  diffusers leaves:
    ``Attention`` = the reference's own vendored copy (VchitectAttention, models/modules/attentions.py:321-638: same
    to_q / to_k / to_v / norm_q / norm_k (qk_norm="layer_norm") / to_out members; its forward handed to the CogVideoX
    processor), ``FeedForward`` = the vendored copy in open_sora_plan_v110_transformer_3d.py:1312-1367, Timesteps /
    TimestepEmbedding restated (load_osp_v110), ``get_3d_sincos_pos_embed`` restated (oracle/cogvideox_oracle.sincos_3d:
    the one leaf of this model that stays unpinned)."""
    if "cogvideox" in _LOADED:
        return _LOADED["cogvideox"]
    O = load_osp_v110()
    A = load().attentions
    from . import cogvideox_oracle as CO

    class Attention(A.VchitectAttention):
        def __init__(self, query_dim, dim_head=64, heads=8, qk_norm=None, eps=1e-5, bias=False, out_bias=True, processor=None, **kw):
            super().__init__(query_dim=query_dim, dim_head=dim_head, heads=heads, qk_norm=qk_norm, eps=eps, bias=bias,
                             out_bias=out_bias, processor=processor, **kw)

        def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, **kw):
            return self.processor(self, hidden_states, encoder_hidden_states=encoder_hidden_states,
                                  attention_mask=attention_mask, **kw)

    class FeedForward(O.FeedForward):
        def __init__(self, dim, dropout=0.0, activation_fn="geglu", final_dropout=False, inner_dim=None, bias=True, **kw):
            assert inner_dim is None and bias, "the vendored copy is the 4x / bias-on configuration"
            super().__init__(dim, dropout=dropout, activation_fn=activation_fn, final_dropout=final_dropout)

    def get_3d_sincos_pos_embed(embed_dim, spatial_size, temporal_size, spatial_interpolation_scale=1.0,
                                temporal_interpolation_scale=1.0):
        return CO.sincos_3d(embed_dim, spatial_size, temporal_size, spatial_interpolation_scale,
                            temporal_interpolation_scale).numpy()

    class Transformer2DModelOutput:
        def __init__(self, sample):
            self.sample = sample

    _mod("diffusers.models.attention", Attention=Attention, FeedForward=FeedForward)
    emb = sys.modules["diffusers.models.embeddings"]
    emb.get_3d_sincos_pos_embed = get_3d_sincos_pos_embed
    _mod("diffusers.models.modeling_outputs", Transformer2DModelOutput=Transformer2DModelOutput)
    sys.modules["diffusers.utils"].is_torch_version = lambda *a, **k: True
    m = importlib.import_module("videosys.models.transformers.cogvideox_transformer_3d")
    _LOADED["cogvideox"] = m
    return m


def build_cogvideox(dtype=torch.float32, **cfg):
    M = load_cogvideox()
    net = M.CogVideoXTransformer3DModel(**cfg).eval().to(dtype)
    net.parallel_manager = SingleRankPM()
    for mod in net.modules():
        if hasattr(mod, "parallel_manager"):
            mod.parallel_manager = SingleRankPM()
    return net


# ---- Vchitect: the reference transformer file imported unmodified; five diffusers leaves restated here ------------------------
class _RefAdaLayerNormZero(nn.Module):
    """diffusers AdaLayerNormZero(embedding_dim) without class embedding: linear(silu(emb)) -> 6 chunks; LayerNorm 1e-6, no affine."""

    def __init__(self, embedding_dim, num_embeddings=None):
        super().__init__()
        self.silu = nn.SiLU()
        self.linear = nn.Linear(embedding_dim, 6 * embedding_dim, bias=True)
        self.norm = nn.LayerNorm(embedding_dim, elementwise_affine=False, eps=1e-6)

    def forward(self, x, timestep=None, class_labels=None, hidden_dtype=None, emb=None):
        emb = self.linear(self.silu(emb))
        shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = emb.chunk(6, dim=1)
        x = self.norm(x) * (1 + scale_msa[:, None]) + shift_msa[:, None]
        return x, gate_msa, shift_mlp, scale_mlp, gate_mlp


class _RefAdaLayerNormContinuous(nn.Module):
    """diffusers AdaLayerNormContinuous(dim, cond_dim, elementwise_affine, eps, bias, norm_type='layer_norm'): scale, shift."""

    def __init__(self, embedding_dim, conditioning_embedding_dim, elementwise_affine=True, eps=1e-5, bias=True, norm_type="layer_norm"):
        super().__init__()
        self.silu = nn.SiLU()
        self.linear = nn.Linear(conditioning_embedding_dim, embedding_dim * 2, bias=bias)
        self.norm = nn.LayerNorm(embedding_dim, eps, elementwise_affine, bias)

    def forward(self, x, conditioning_embedding):
        emb = self.linear(self.silu(conditioning_embedding).to(x.dtype))
        scale, shift = torch.chunk(emb, 2, dim=1)
        return self.norm(x) * (1 + scale)[:, None, :] + shift[:, None, :]


class _RefCombinedTimestepTextProj(nn.Module):
    """diffusers CombinedTimestepTextProjEmbeddings(embedding_dim, pooled_projection_dim)."""

    def __init__(self, embedding_dim, pooled_projection_dim):
        super().__init__()
        self.time_proj = _RefTimesteps(num_channels=256, flip_sin_to_cos=True, downscale_freq_shift=0)
        self.timestep_embedder = _RefTimestepEmbedding(in_channels=256, time_embed_dim=embedding_dim)
        self.text_embedder = _RefTimestepEmbedding(pooled_projection_dim, embedding_dim)  # PixArtAlphaTextProjection(act_fn="silu")

    def forward(self, timestep, pooled_projection):
        timesteps_emb = self.timestep_embedder(self.time_proj(timestep).to(dtype=pooled_projection.dtype))
        return timesteps_emb + self.text_embedder(pooled_projection)


class _RefPatchEmbedSD3(nn.Module):
    """diffusers PatchEmbed with pos_embed_max_size (SD3): conv, flatten, + the centre crop of a max-size sin-cos table."""

    def __init__(self, height=224, width=224, patch_size=16, in_channels=3, embed_dim=768, pos_embed_max_size=None, **_):
        super().__init__()
        import numpy as np

        self.proj = nn.Conv2d(in_channels, embed_dim, kernel_size=(patch_size, patch_size), stride=patch_size, bias=True)
        self.patch_size, self.pos_embed_max_size = patch_size, pos_embed_max_size
        base = height // patch_size
        g = np.arange(pos_embed_max_size, dtype=np.float32) / (pos_embed_max_size / base)
        grid = np.stack(np.meshgrid(g, g), axis=0).reshape([2, 1, pos_embed_max_size, pos_embed_max_size])

        def one(dim, pos):
            omega = 1.0 / 10000 ** (np.arange(dim // 2, dtype=np.float64) / (dim / 2.0))
            out = np.einsum("m,d->md", pos.reshape(-1), omega)
            return np.concatenate([np.sin(out), np.cos(out)], axis=1)

        pe = np.concatenate([one(embed_dim // 2, grid[0]), one(embed_dim // 2, grid[1])], axis=1)
        self.register_buffer("pos_embed", torch.from_numpy(pe).float().unsqueeze(0), persistent=True)

    def forward(self, latent):
        h, w = latent.shape[-2] // self.patch_size, latent.shape[-1] // self.patch_size
        latent = self.proj(latent).flatten(2).transpose(1, 2)
        m = self.pos_embed_max_size
        top, left = (m - h) // 2, (m - w) // 2
        pe = self.pos_embed.reshape(1, m, m, -1)[:, top : top + h, left : left + w, :].reshape(1, -1, self.pos_embed.shape[-1])
        return (latent + pe).to(latent.dtype)


def load_vchitect():
    """models/transformers/vchitect_transformer_3d.py imported unmodified (JointTransformerBlock, FeedForward,
    VchitectXLTransformerModel incl. precompute_freqs_cis and forward) on top of the reference's own VchitectAttention +
    processor; the five diffusers leaf classes above are restated from their published semantics."""
    if "vchitect" in _LOADED:
        return _LOADED["vchitect"]
    load_osp_v110()  # shared stubs
    ph = lambda name: type(name, (), {})  # noqa: E731
    _mod("diffusers.loaders", FromOriginalModelMixin=ph("FromOriginalModelMixin"), PeftAdapterMixin=ph("PeftAdapterMixin"))
    emb = sys.modules["diffusers.models.embeddings"]
    emb.CombinedTimestepTextProjEmbeddings = _RefCombinedTimestepTextProj
    emb.PatchEmbed = _RefPatchEmbedSD3
    norm = sys.modules["diffusers.models.normalization"]
    norm.AdaLayerNormContinuous = _RefAdaLayerNormContinuous
    norm.AdaLayerNormZero = _RefAdaLayerNormZero
    _mod("diffusers.models.transformers")
    _mod("diffusers.models.transformers.transformer_2d",
         Transformer2DModelOutput=type("Transformer2DModelOutput", (), {"__init__": lambda s, sample: setattr(s, "sample", sample)}))
    sys.modules["diffusers.utils"].unscale_lora_layers = lambda *a, **k: None
    m = importlib.import_module("videosys.models.transformers.vchitect_transformer_3d")
    _LOADED["vchitect"] = m
    return m


def build_vchitect(dtype=torch.float32, **cfg):
    M = load_vchitect()
    net = M.VchitectXLTransformerModel(**cfg).eval().to(dtype)
    net.parallel_manager = SingleRankPM()
    for mod in net.modules():
        if hasattr(mod, "parallel_manager"):
            mod.parallel_manager = SingleRankPM()
    return net


def load_osp_v120():
    """The reference's models/transformers/open_sora_plan_v120_transformer_3d.py (RoPE3D, PatchEmbed2D, Attention +
    AttnProcessor2_0, BasicTransformerBlock, OpenSoraT2V), imported unmodified.  diffusers leaves: ``Attention`` (base class)
    = the reference's vendored copy in the v1.1.0 file, ``FeedForward`` / ``AdaLayerNormSingle`` / ``PixArtAlphaTextProjection``
    = the vendored copies there (FeedForward, AdaLayerNormSingle, CaptionProjection), plus the three restated leaves."""
    if "osp_v120" in _LOADED:
        return _LOADED["osp_v120"]
    O = load_osp_v110()

    class FeedForward(O.FeedForward):
        def __init__(self, dim, dropout=0.0, activation_fn="geglu", final_dropout=False, inner_dim=None, bias=True, **kw):
            assert inner_dim is None and bias, "the vendored copy is the 4x / bias-on configuration"
            super().__init__(dim, dropout=dropout, activation_fn=activation_fn, final_dropout=final_dropout)

    class PixArtAlphaTextProjection(O.CaptionProjection):
        def __init__(self, in_features, hidden_size, **kw):
            super().__init__(in_features, hidden_size)
            del self._buffers["y_embedding"]

    ph = lambda name: type(name, (nn.Module,), {})  # noqa: E731
    _mod("diffusers.models.attention", FeedForward=FeedForward, GatedSelfAttentionDense=ph("GatedSelfAttentionDense"),
         Attention=sys.modules["diffusers.models.attention"].Attention if hasattr(sys.modules.get("diffusers.models.attention"), "Attention") else object)
    sys.modules["diffusers.models.attention_processor"].Attention = O.Attention
    emb = sys.modules["diffusers.models.embeddings"]
    emb.PixArtAlphaTextProjection = PixArtAlphaTextProjection
    norm = sys.modules["diffusers.models.normalization"]
    norm.AdaLayerNormSingle = O.AdaLayerNormSingle
    if not hasattr(norm, "AdaLayerNormContinuous"):
        norm.AdaLayerNormContinuous = ph("AdaLayerNormContinuous")
    sys.modules["diffusers.utils"].is_torch_version = lambda *a, **k: True
    _mod("diffusers.pipelines")
    _mod("diffusers.pipelines.pipeline_utils", DiffusionPipeline=type("DiffusionPipeline", (), {"__init__": lambda s: None}))
    m = importlib.import_module("videosys.models.transformers.open_sora_plan_v120_transformer_3d")
    _LOADED["osp_v120"] = m
    return m


def build_osp_v120(dtype=torch.float32, **cfg):
    M = load_osp_v120()
    net = M.OpenSoraT2V(**cfg).eval().to(dtype)
    net.parallel_manager = SingleRankPM()
    for mod in net.modules():
        if hasattr(mod, "parallel_manager"):
            mod.parallel_manager = SingleRankPM()
    return net
