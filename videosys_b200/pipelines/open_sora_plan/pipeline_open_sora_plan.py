"""Open-Sora-Plan pipeline surface (mirror of videosys/pipelines/open_sora_plan/pipeline_open_sora_plan.py:
OpenSoraPlanV110PABConfig :41-100, OpenSoraPlanV120PABConfig :103-120, OpenSoraPlanConfig :123-226,
OpenSoraPlanPipeline.generate :962-1180) around the native transformer.

Version v110 (``LatteT2V``, 65 or 221 frames at 512 x 512, head_dim 72): CFG batch of 2, PNDM steps (incl. its Runge-Kutta
warm-up: the transformer is evaluated at every entry of ``scheduler.timesteps``), learned-sigma split, PAB with the MLP skip.
Version v120 (``OpenSoraT2V``, 29 or 93 frames at 480p / 720p, head_dim 96, 3-D RoPE): ancestral Euler steps (the latent is
scaled by the scheduler before every forward, :1097), PAB with the spatial and the cross gate; its attention runs on the
warp-level kernel of csrc/attn_mma.cu (head_dim 64 / 72 run on csrc/attn_wgmma.cu).

Opt-in through ``OpenSoraPlanConfig(vae=...)``: the causal-VAE decode tail (:1168-1191) on the native decoder of the
version (models/autoencoders/autoencoder_kl_open_sora_plan.py), tiled with the reference's sizes when ``enable_tiling``
(:309-315), then ``((v / 2 + 0.5).clamp(0, 1) * 255).to(uint8)`` as ``[B, T, H, W, 3]``, cut to the requested frames and
size.  Out of scope as for the other pipelines (SURVEY.md 2.1): the T5 encoder -- pass ``prompt_embeds`` (+ masks) or a
``text_encoder_fn``.  Without a ``vae`` or a ``vae_decode_fn`` the LATENTS are returned.  dtype fp16 as the reference (:262).
"""
import math
import zlib
from typing import Callable, Optional

import torch

from ...core.pab.pab_mgr import PABConfig, enable_pab, set_pab_manager, update_steps
from ...models.transformers.open_sora_plan_v110_transformer_3d import LatteT2V
from ...models.transformers.open_sora_plan_v120_transformer_3d import OpenSoraT2V
from ...schedulers.scheduling_euler_ancestral import EulerAncestralDiscreteScheduler
from ...schedulers.scheduling_pndm import PNDMScheduler
from .._common import ParallelPipelineMixin
from ..open_sora.pipeline_open_sora import VideoSysPipelineOutput

_V110_MLP = {k: {"block": [0, 1, 2, 3, 4, 5, 6], "skip_count": 2} for k in (738, 714, 690, 666, 642, 618, 594, 570, 546, 522, 498, 474, 450, 426)}


class OpenSoraPlanV110PABConfig(PABConfig):
    def __init__(self, spatial_broadcast=True, spatial_threshold=(100, 850), spatial_range=2, temporal_broadcast=True,
                 temporal_threshold=(100, 850), temporal_range=4, cross_broadcast=True, cross_threshold=(100, 850),
                 cross_range=6, mlp_broadcast=True, mlp_spatial_broadcast_config=None, mlp_temporal_broadcast_config=None):
        super().__init__(
            spatial_broadcast=spatial_broadcast, spatial_threshold=list(spatial_threshold), spatial_range=spatial_range,
            temporal_broadcast=temporal_broadcast, temporal_threshold=list(temporal_threshold), temporal_range=temporal_range,
            cross_broadcast=cross_broadcast, cross_threshold=list(cross_threshold), cross_range=cross_range,
            mlp_broadcast=mlp_broadcast,
            mlp_spatial_broadcast_config=dict(_V110_MLP) if mlp_spatial_broadcast_config is None else mlp_spatial_broadcast_config,
            mlp_temporal_broadcast_config=dict(_V110_MLP) if mlp_temporal_broadcast_config is None else mlp_temporal_broadcast_config)


class OpenSoraPlanV120PABConfig(PABConfig):
    def __init__(self, spatial_broadcast=True, spatial_threshold=(100, 850), spatial_range=2, cross_broadcast=True,
                 cross_threshold=(100, 850), cross_range=6):
        super().__init__(spatial_broadcast=spatial_broadcast, spatial_threshold=list(spatial_threshold),
                         spatial_range=spatial_range, cross_broadcast=cross_broadcast, cross_threshold=list(cross_threshold),
                         cross_range=cross_range)


class OpenSoraPlanConfig:
    def __init__(self, version: str = "v120", transformer_type: str = "29x480p", transformer: str = None, text_encoder: str = None,
                 num_gpus: int = 1, cpu_offload: bool = False, enable_tiling: bool = True, tile_overlap_factor: float = 0.25,
                 enable_pab: bool = False, pab_config: PABConfig = None, transformer_config: Optional[dict] = None,
                 state_dict=None, text_encoder_fn: Optional[Callable] = None, vae_decode_fn: Optional[Callable] = None,
                 vae=None):
        self.pipeline_cls = OpenSoraPlanPipeline
        assert version in ["v110", "v120"], f"Unknown Open-Sora-Plan version: {version}"
        self.version, self.transformer_type = version, transformer_type
        if version == "v110":
            assert transformer_type in ["65x512x512", "221x512x512"]
        else:
            assert transformer_type in ["93x480p", "93x720p", "29x480p", "29x720p"]
        self.num_frames = int(transformer_type.split("x")[0])
        self.text_encoder = text_encoder or ("DeepFloyd/t5-v1_1-xxl" if version == "v110" else "google/mt5-xxl")
        self.transformer = transformer or f"LanguageBind/Open-Sora-Plan-{'v1.1.0' if version == 'v110' else 'v1.2.0'}"
        self.num_gpus, self.cpu_offload = num_gpus, cpu_offload
        self.enable_tiling, self.tile_overlap_factor = enable_tiling, tile_overlap_factor
        self.enable_pab = enable_pab
        if enable_pab and pab_config is None:
            pab_config = OpenSoraPlanV110PABConfig() if version == "v110" else OpenSoraPlanV120PABConfig()
        self.pab_config = pab_config
        # native build extras: architecture / weights / out-of-scope stages supplied by the caller
        self.transformer_config, self.state_dict = transformer_config, state_dict
        self.text_encoder_fn, self.vae_decode_fn = text_encoder_fn, vae_decode_fn
        # native VAE decoder: a local snapshot directory (its root or its vae/ folder) or a decoder instance of the version
        self.vae = vae


class OpenSoraPlanPipeline(ParallelPipelineMixin):
    vae_scale_factor = (4, 8, 8)  # the causal VAE's (t, h, w) compression

    def __init__(self, config: OpenSoraPlanConfig, device=None, dtype: torch.dtype = torch.float16):
        if not torch.cuda.is_available():
            raise RuntimeError("videosys_b200 pipelines need an sm_90a GPU (no CPU path)")
        import os

        self._config, self._dtype = config, dtype
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        tc = config.transformer_config
        cls = LatteT2V if config.version == "v110" else OpenSoraT2V
        if tc is None and config.state_dict is None and os.path.isdir(str(config.transformer)):
            self.transformer = cls.from_pretrained(config.transformer, subfolder=config.transformer_type).to(dtype)
        elif config.version == "v110":
            self.transformer = LatteT2V(**(tc or dict(video_length=self.latent_frames(config.num_frames)))).to(dtype)
        else:
            hw = (60, 80) if config.transformer_type.endswith("480p") else (90, 160)  # latent height x width of 480p / 720p
            self.transformer = OpenSoraT2V(**(tc or dict(sample_size=hw, sample_size_t=self.latent_frames(config.num_frames)))).to(dtype)
        if config.state_dict is not None:
            self.transformer.load_state_dict(config.state_dict)
        self.transformer = self.transformer.to(self._device).eval()
        self.scheduler = PNDMScheduler() if config.version == "v110" else EulerAncestralDiscreteScheduler()
        self.vae = self._load_vae()
        if config.enable_pab:
            set_pab_manager(config.pab_config)
        self._set_parallel()

    def _load_vae(self):
        """The native decoder of ``config.vae`` in the pipeline dtype, with the reference's tiling settings (:309-315)."""
        import os

        from ...models.autoencoders.autoencoder_kl_open_sora_plan import decoder_class

        cls = decoder_class(self._config.version)
        v = self._config.vae
        if v is None:
            return None
        if not isinstance(v, cls):
            v = str(v)
            v = cls.from_pretrained(v, subfolder="vae" if os.path.isdir(os.path.join(v, "vae")) else None)
        v = v.to(self._dtype).to(self._device).eval()
        if self._config.enable_tiling:
            v.enable_tiling()
            v.tile_overlap_factor = self._config.tile_overlap_factor
            v.tile_sample_min_size = 512
            v.tile_latent_min_size = 64
            v.tile_sample_min_size_t = 29
            v.tile_latent_min_size_t = 8
        return v

    def decode_latents(self, latents):
        """Reference decode_latents (:1184-1191) with CausalVAEModelWrapper.decode: latents [B, C, T, h, w] ->
        uint8 [B, T', H, W, 3]."""
        video = self.vae.decode(latents.to(self.vae.dtype) / 0.18215).permute(0, 2, 1, 3, 4)  # b t c h w
        return ((video / 2.0 + 0.5).clamp(0, 1) * 255).to(dtype=torch.uint8).cpu().permute(0, 1, 3, 4, 2).contiguous()

    @classmethod
    def latent_frames(cls, num_frames: int) -> int:
        """reference prepare_latents :893-897."""
        f = cls.vae_scale_factor[0]
        return math.ceil((int(num_frames) - 1) / f) + 1 if int(num_frames) % 2 == 1 else math.ceil(int(num_frames) / f)

    def _embeds(self, prompt, negative_prompt, L=300):
        cfg = self.transformer.config
        if self._config.text_encoder_fn is not None:
            return self._config.text_encoder_fn(prompt, negative_prompt)
        g = torch.Generator(device="cpu").manual_seed(zlib.crc32(str(prompt).encode()))
        n = 20 + zlib.crc32(str(prompt).encode()) % 60  # a synthetic caption length: the rest is tokenizer padding
        mask = (torch.arange(L)[None] < n).to(torch.int64)
        nmask = (torch.arange(L)[None] < 1).to(torch.int64)  # the empty negative prompt keeps its end-of-sequence token
        return (torch.randn(1, L, cfg.caption_channels, generator=g), mask, torch.randn(1, L, cfg.caption_channels, generator=g), nmask)

    @torch.no_grad()
    def generate(self, prompt=None, negative_prompt: str = "", num_inference_steps: int = 150, guidance_scale: float = 7.5,
                 num_images_per_prompt: int = 1, eta: float = 0.0, seed: int = -1, generator=None, latents=None,
                 prompt_embeds=None, prompt_attention_mask=None, negative_prompt_embeds=None,
                 negative_prompt_attention_mask=None, output_type: str = "pil", return_dict: bool = True, callback=None,
                 callback_steps: int = 1, clean_caption: bool = True, mask_feature: bool = True,
                 enable_temporal_attentions: bool = True, verbose: bool = True, max_sequence_length: int = 300,
                 height: int = 512, width: int = 512):
        """height / width follow the transformer's sample size in the reference (:1005-1007: 512 x 512 for v110, the 480p / 720p
        grid for v120; the arguments are used by v110 only, so that the tests can run a small model)."""
        v120 = self._config.version == "v120"
        if v120:
            height = self.transformer.config.sample_size[0] * self.vae_scale_factor[1]
            width = self.transformer.config.sample_size[1] * self.vae_scale_factor[2]
        update_steps(num_inference_steps)
        self.transformer.reset_pab_state()
        self._maybe_seed(seed)
        dev, dt = self._device, self._dtype
        if prompt_embeds is None:
            prompt_embeds, prompt_attention_mask, negative_prompt_embeds, negative_prompt_attention_mask = self._embeds(
                prompt, negative_prompt, max_sequence_length)
        do_cfg = guidance_scale > 1.0
        if prompt_attention_mask is None:  # caller-supplied embeddings without masks: every token is valid
            prompt_attention_mask = torch.ones(prompt_embeds.shape[0], prompt_embeds.shape[-2], dtype=torch.int64)
        if do_cfg and negative_prompt_attention_mask is None:
            negative_prompt_attention_mask = torch.ones(negative_prompt_embeds.shape[0], negative_prompt_embeds.shape[-2], dtype=torch.int64)
        pe, pm = prompt_embeds.to(dev, dt), prompt_attention_mask
        if do_cfg:  # reference encode_prompt: [negative, positive]
            pe = torch.cat([negative_prompt_embeds.to(dev, dt), pe], dim=0)
            pm = torch.cat([negative_prompt_attention_mask, prompt_attention_mask], dim=0)
        self.scheduler.set_timesteps(num_inference_steps, dev)
        ts = [(float(v) if v120 else int(v)) for v in self.scheduler.timesteps.tolist()]
        cin = self.transformer.config.in_channels
        if self._config.transformer_config is None:
            Fr = self.latent_frames(self._config.num_frames)
        else:
            Fr = self.transformer.config.sample_size_t if v120 else self.transformer.video_length
        if latents is None:
            latents = torch.randn(prompt_embeds.shape[0], cin, Fr, height // self.vae_scale_factor[1],
                                  width // self.vae_scale_factor[2], device=dev, dtype=dt)
        lat = latents.to(dev, dt) * self.scheduler.init_noise_sigma
        for t in ts:
            inp = torch.cat([lat] * 2) if do_cfg else lat
            if v120:
                inp = self.scheduler.scale_model_input(inp, t).to(dt)
            tt = torch.full((inp.shape[0],), t, device=dev, dtype=torch.float32 if v120 else torch.int64)
            noise = self.transformer(inp, timestep=tt, all_timesteps=ts, encoder_hidden_states=pe.unsqueeze(1),
                                     added_cond_kwargs={"resolution": None, "aspect_ratio": None},
                                     enable_temporal_attentions=enable_temporal_attentions,
                                     encoder_attention_mask=pm.unsqueeze(1), return_dict=False,
                                     ts_int=int(t) if enable_pab() else None)[0]
            if do_cfg:
                un, tx = noise.chunk(2)
                noise = un + guidance_scale * (tx - un)
            if self.transformer.config.out_channels // 2 == cin:  # learned sigma: keep the mean prediction (:1150-1153)
                noise = noise.chunk(2, dim=1)[0]
            lat = self.scheduler.step(noise, t, lat)[0].to(dt)
        if self._config.vae_decode_fn is not None and output_type != "latents":
            video = self._config.vae_decode_fn(lat)
        elif getattr(self, "vae", None) is not None and output_type != "latents":
            video = self.decode_latents(lat)[:, :self._config.num_frames, :height, :width]
        else:
            video = lat.float().cpu()  # latents: the VAE is out of scope
        return VideoSysPipelineOutput(video=video) if return_dict else (video,)
