"""Latte pipeline surface (mirror of videosys/pipelines/latte/pipeline_latte.py: LattePABConfig :35-76, LatteConfig
:127-160, LattePipeline.generate :675-905) around the native LatteT2V.

In scope: the config classes, ``generate()``'s signature, the CFG + DDIM loop (:815-873, learned-sigma split :864-868),
the denoiser, and -- opt-in through ``LatteConfig(vae=...)`` -- the VAE decode tail (:884-946) on a native decoder: the
temporal decoder (models/autoencoders/autoencoder_kl_temporal_decoder.py, ``vae_temporal_decoder/``) or, with
``enable_vae_temporal_decoder=False``, the image VAE (models/autoencoders/autoencoder_kl.py, ``vae/``), as the reference
loads them (:211-217).  Out of scope as for the other pipelines (SURVEY.md 2.1): T5 encoder, caption cleaning -- pass
``prompt_embeds`` / ``negative_prompt_embeds`` or a ``text_encoder_fn``.  Without a ``vae`` or a ``vae_decode_fn`` the
LATENTS are returned.  dtype fp16 as the reference (:201).  Latte generates 16 frames at 512 x 512 (:764-766).
"""
import os
import zlib
from typing import Callable, Optional

import torch

from ...core.pab.pab_mgr import PABConfig, enable_pab, set_pab_manager, update_steps
from ...models.transformers.latte_transformer_3d import LatteT2V
from ...schedulers.scheduling_ddim import DDIMScheduler
from ...models.autoencoders.autoencoder_kl import AutoencoderKL
from ...models.autoencoders.autoencoder_kl_temporal_decoder import AutoencoderKLTemporalDecoder
from .._common import ParallelPipelineMixin, decode_image_frames
from ..open_sora.pipeline_open_sora import VideoSysPipelineOutput

_MLP_CFG = {k: {"block": [0, 1, 2, 3, 4], "skip_count": 2} for k in (720, 640, 560, 480, 400)}


class LattePABConfig(PABConfig):
    def __init__(self, spatial_broadcast=True, spatial_threshold=(100, 800), spatial_range=2, temporal_broadcast=True,
                 temporal_threshold=(100, 800), temporal_range=3, cross_broadcast=True, cross_threshold=(100, 800),
                 cross_range=6, mlp_broadcast=True, mlp_spatial_broadcast_config=None, mlp_temporal_broadcast_config=None):
        super().__init__(
            spatial_broadcast=spatial_broadcast, spatial_threshold=list(spatial_threshold), spatial_range=spatial_range,
            temporal_broadcast=temporal_broadcast, temporal_threshold=list(temporal_threshold), temporal_range=temporal_range,
            cross_broadcast=cross_broadcast, cross_threshold=list(cross_threshold), cross_range=cross_range,
            mlp_broadcast=mlp_broadcast,
            mlp_spatial_broadcast_config=dict(_MLP_CFG) if mlp_spatial_broadcast_config is None else mlp_spatial_broadcast_config,
            mlp_temporal_broadcast_config=dict(_MLP_CFG) if mlp_temporal_broadcast_config is None else mlp_temporal_broadcast_config,
        )


class LatteConfig:
    def __init__(self, model_path: str = "maxin-cn/Latte-1", num_gpus: int = 1, enable_vae_temporal_decoder: bool = True,
                 beta_start: float = 0.0001, beta_end: float = 0.02, beta_schedule: str = "linear",
                 variance_type: str = "learned_range", enable_pab: bool = False, pab_config=None,
                 transformer_config: Optional[dict] = None, state_dict=None, text_encoder_fn: Optional[Callable] = None,
                 vae_decode_fn: Optional[Callable] = None, vae=None):
        self.model_path = model_path
        self.pipeline_cls = LattePipeline
        self.num_gpus = num_gpus
        self.enable_vae_temporal_decoder = enable_vae_temporal_decoder
        self.beta_start, self.beta_end, self.beta_schedule, self.variance_type = beta_start, beta_end, beta_schedule, variance_type
        self.enable_pab = enable_pab
        self.pab_config = pab_config if pab_config is not None else LattePABConfig()
        # native build extras: architecture / weights / out-of-scope stages supplied by the caller
        self.transformer_config = transformer_config
        self.state_dict = state_dict
        self.text_encoder_fn = text_encoder_fn
        self.vae_decode_fn = vae_decode_fn
        # native VAE decoder: a local snapshot root, or an AutoencoderKLTemporalDecoder / AutoencoderKL instance
        self.vae = vae


class LattePipeline(ParallelPipelineMixin):
    vae_scale_factor = 8
    vae = None  # the native VAE decoder (_load_vae); without one generate returns the latents
    decode_chunk_size = 14  # frames per temporal-decoder pass (:931)

    def __init__(self, config: LatteConfig, device=None, dtype: torch.dtype = torch.float16):
        if not torch.cuda.is_available():
            raise RuntimeError("videosys_b200 pipelines need an sm_90a GPU (no CPU path)")
        self._config = config
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._dtype = dtype
        import os

        if config.transformer_config is None and config.state_dict is None and os.path.isdir(str(config.model_path)):
            self.transformer = LatteT2V.from_pretrained(config.model_path, subfolder="transformer", video_length=16).to(dtype)
        else:
            self.transformer = LatteT2V(**(config.transformer_config or {})).to(dtype)
        if config.state_dict is not None:
            self.transformer.load_state_dict(config.state_dict)
        self.transformer = self.transformer.to(self._device).eval()
        self.scheduler = DDIMScheduler(beta_start=config.beta_start, beta_end=config.beta_end, beta_schedule=config.beta_schedule,
                                       variance_type=config.variance_type, clip_sample=False)
        self.vae = self._load_vae()
        if config.enable_pab:
            set_pab_manager(config.pab_config)
        self._set_parallel()

    def _load_vae(self):
        """The native decoder of ``config.vae`` in the pipeline dtype: an instance as it is, a snapshot root through its
        ``vae_temporal_decoder/`` or ``vae/`` folder as enable_vae_temporal_decoder picks (:211-217)."""
        v = self._config.vae
        if v is None:
            return None
        if not isinstance(v, (AutoencoderKLTemporalDecoder, AutoencoderKL)):
            if self._config.enable_vae_temporal_decoder:
                v = AutoencoderKLTemporalDecoder.from_pretrained(os.fspath(v), subfolder="vae_temporal_decoder")
            else:
                v = AutoencoderKL.from_pretrained(os.fspath(v), subfolder="vae")
        return v.to(self._dtype).to(self._device).eval()

    @staticmethod
    def _frames(latents):
        """einops "b c f h w -> (b f) c h w"."""
        b, c, f, h, w = latents.shape
        return latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)

    def _decode_frames(self, z, num_frames=None):
        """z [N, C, h, w] through the decoder: the temporal decoder in chunks of ``num_frames`` frames decoded as one video
        each, the image VAE frame by frame (several per pass: each frame is its own GroupNorm sample)."""
        if num_frames is None:
            return decode_image_frames(self.vae, z)
        return torch.cat([self.vae.decode(z[i:i + num_frames], num_frames=z[i:i + num_frames].shape[0]).sample
                          for i in range(0, z.shape[0], num_frames)])

    def decode_latents_image(self, latents):
        """Reference :904-914: float [B, F, 3, H, W] in [0, 1].  The temporal decoder takes each frame as a video of
        one frame."""
        b, _, f = latents.shape[:3]
        z = self._frames(1 / self.vae.config.scaling_factor * latents)
        video = self._decode_frames(z, 1 if isinstance(self.vae, AutoencoderKLTemporalDecoder) else None)
        return (video.view(b, f, *video.shape[1:]) / 2.0 + 0.5).clamp(0, 1)

    def decode_video(self, latents):
        """Reference :916-922 (image VAE, per frame) or :927-943 (temporal decoder: the flattened frames in chunks of
        decode_chunk_size, a chunk possibly holding the end of one sample and the start of the next, decoded as one
        video as the reference does): float [B, F, H, W, 3], before the uint8 conversion."""
        b, _, f = latents.shape[:3]
        z = self._frames(1 / self.vae.config.scaling_factor * latents)
        video = self._decode_frames(z, self.decode_chunk_size if isinstance(self.vae, AutoencoderKLTemporalDecoder) else None)
        return video.view(b, f, *video.shape[1:]).permute(0, 1, 3, 4, 2)

    @staticmethod
    def to_uint8(video):
        """Reference :923-924 / :944-945: uint8 on the CPU."""
        return ((video / 2.0 + 0.5).clamp(0, 1) * 255).to(dtype=torch.uint8).cpu().contiguous()

    def _embeds(self, prompt, negative_prompt, L=120):
        cfg = self.transformer.config
        if self._config.text_encoder_fn is not None:
            return self._config.text_encoder_fn(prompt, negative_prompt)
        g = torch.Generator(device="cpu").manual_seed(zlib.crc32(str(prompt).encode()))
        return torch.randn(1, L, cfg.caption_channels, generator=g), torch.randn(1, L, cfg.caption_channels, generator=g)

    @torch.no_grad()
    def generate(self, prompt=None, negative_prompt: str = "", num_inference_steps: int = 50, guidance_scale: float = 7.5,
                 num_images_per_prompt: int = 1, eta: float = 0.0, seed: int = -1, generator=None, latents=None,
                 prompt_embeds=None, negative_prompt_embeds=None, output_type: str = "pil", return_dict: bool = True,
                 callback=None, callback_steps: int = 1, clean_caption: bool = True, mask_feature: bool = True,
                 enable_temporal_attentions: bool = True, verbose: bool = True, video_length: int = 16, height: int = 512,
                 width: int = 512):
        """video_length / height / width are fixed to 16 / 512 / 512 by the reference (:764-766); they are arguments here so
        that the tests can run a small model."""
        update_steps(num_inference_steps)
        self.transformer.reset_pab_state()
        self._maybe_seed(seed)
        dev, dt = self._device, self._dtype
        if prompt_embeds is None:
            prompt_embeds, negative_prompt_embeds = self._embeds(prompt, negative_prompt)
        do_cfg = guidance_scale > 1.0
        pe = prompt_embeds.to(dev, dt)
        if do_cfg:
            pe = torch.cat([negative_prompt_embeds.to(dev, dt), pe], dim=0)
        self.scheduler.set_timesteps(num_inference_steps, dev)
        ts = [int(v) for v in self.scheduler.timesteps.tolist()]
        cin = self.transformer.config.in_channels
        if latents is None:
            latents = torch.randn(prompt_embeds.shape[0], cin, video_length, height // self.vae_scale_factor,
                                  width // self.vae_scale_factor, device=dev, dtype=dt)
        lat = latents.to(dev, dt) * self.scheduler.init_noise_sigma
        for t in ts:
            inp = torch.cat([lat] * 2) if do_cfg else lat
            tt = torch.full((inp.shape[0],), t, device=dev, dtype=torch.int64)
            noise = self.transformer(inp, timestep=tt, all_timesteps=ts, encoder_hidden_states=pe,
                                     added_cond_kwargs={"resolution": None, "aspect_ratio": None},
                                     enable_temporal_attentions=enable_temporal_attentions, return_dict=False,
                                     ts_int=t if enable_pab() else None)[0]
            if do_cfg:
                un, tx = noise.chunk(2)
                noise = un + guidance_scale * (tx - un)
            if self.transformer.config.out_channels // 2 == cin:  # learned sigma: keep the mean prediction (:864-868)
                noise = noise.chunk(2, dim=1)[0]
            lat = self.scheduler.step(noise, t, lat, eta=eta)[0]
        if self._config.vae_decode_fn is not None and output_type != "latents":
            video = self._config.vae_decode_fn(lat)
        elif self.vae is not None and output_type != "latents":  # :884-891
            video = self.decode_latents_image(lat) if lat.shape[2] == 1 else self.to_uint8(self.decode_video(lat))
        else:
            video = lat.float().cpu()  # latents
        return VideoSysPipelineOutput(video=video) if return_dict else (video,)
