"""Vchitect-2.0 pipeline surface (mirror of videosys/pipelines/vchitect/pipeline_vchitect.py: VchitectPABConfig :30-53,
VchitectConfig :56-127, VchitectXLPipeline.generate :712-1009) around the native VchitectXLTransformerModel.

In scope: the config classes, ``generate()``'s signature, the denoising loop as the reference runs it (:916-954: the
unconditional and the text branch are two batch-1 forwards, the guidance scale follows the cosine ramp of :943-945,
flow-match Euler update), the denoiser, and -- opt-in through ``VchitectConfig(vae=...)`` -- the VAE decode tail
(:980-986) on the native image decoder (models/autoencoders/autoencoder_kl.py, the snapshot's ``vae/`` folder, :214-215)
with diffusers' ``VaeImageProcessor.postprocess`` per frame (pipelines/_common.py).  Out of scope as for the other
pipelines (SURVEY.md 2.1): the three text encoders -- pass ``prompt_embeds`` / ``pooled_prompt_embeds`` (and the
negative pair) or a ``text_encoder_fn``.  Without a ``vae`` or a ``vae_decode_fn`` the LATENTS ``[1, frames, C, H/8,
W/8]`` are returned.  dtype bf16 as the reference (:186).
"""
import math
import os
import zlib
from typing import Callable, Optional

import torch

from ...core.pab.pab_mgr import PABConfig, enable_pab, set_pab_manager, update_steps
from ...models.transformers.vchitect_transformer_3d import VchitectXLTransformerModel
from ...schedulers.scheduling_flow_match_euler import FlowMatchEulerDiscreteScheduler
from ...models.autoencoders.autoencoder_kl import AutoencoderKL
from .._common import ParallelPipelineMixin, decode_image_frames, postprocess_frames
from ..open_sora.pipeline_open_sora import VideoSysPipelineOutput


class VchitectPABConfig(PABConfig):
    def __init__(self, spatial_broadcast=True, spatial_threshold=(100, 800), spatial_range=2, temporal_broadcast=True,
                 temporal_threshold=(100, 800), temporal_range=4, cross_broadcast=True, cross_threshold=(100, 800),
                 cross_range=6):
        super().__init__(
            spatial_broadcast=spatial_broadcast, spatial_threshold=list(spatial_threshold), spatial_range=spatial_range,
            temporal_broadcast=temporal_broadcast, temporal_threshold=list(temporal_threshold), temporal_range=temporal_range,
            cross_broadcast=cross_broadcast, cross_threshold=list(cross_threshold), cross_range=cross_range)


class VchitectConfig:
    def __init__(self, model_path: str = "Vchitect/Vchitect-2.0-2B", num_gpus: int = 1, cpu_offload: bool = False,
                 enable_pab: bool = False, pab_config=None, transformer_config: Optional[dict] = None, state_dict=None,
                 scheduler_shift: float = 3.0, text_encoder_fn: Optional[Callable] = None,
                 vae_decode_fn: Optional[Callable] = None, vae=None):
        self.model_path = model_path
        self.pipeline_cls = VchitectXLPipeline
        self.num_gpus = num_gpus
        self.cpu_offload = cpu_offload
        self.enable_pab = enable_pab
        self.pab_config = pab_config if pab_config is not None else VchitectPABConfig()
        # native build extras: architecture / weights / scheduler shift (the HF scheduler_config.json is not in the tree) /
        # out-of-scope stages supplied by the caller
        self.transformer_config = transformer_config
        self.state_dict = state_dict
        self.scheduler_shift = scheduler_shift
        self.text_encoder_fn = text_encoder_fn
        self.vae_decode_fn = vae_decode_fn
        # native VAE decoder: a local snapshot root (its vae/ folder is read) or an AutoencoderKL instance
        self.vae = vae


class VchitectXLPipeline(ParallelPipelineMixin):
    vae_scale_factor = 8
    vae = None  # the native VAE decoder (_load_vae); without one generate returns the latents

    def __init__(self, config: VchitectConfig, device=None, dtype: torch.dtype = torch.bfloat16):
        if not torch.cuda.is_available():
            raise RuntimeError("videosys_b200 pipelines need an sm_90a GPU (no CPU path)")
        import os

        self._config = config
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._dtype = dtype
        if config.transformer_config is None and config.state_dict is None and os.path.isdir(str(config.model_path)):
            self.transformer = VchitectXLTransformerModel.from_pretrained(config.model_path, subfolder="transformer").to(dtype)
        else:
            self.transformer = VchitectXLTransformerModel(**(config.transformer_config or {})).to(dtype)
        if config.state_dict is not None:
            self.transformer.load_state_dict(config.state_dict)
        self.transformer = self.transformer.to(self._device).eval()
        self.scheduler = FlowMatchEulerDiscreteScheduler(shift=config.scheduler_shift)
        self.vae = self._load_vae()
        if config.enable_pab:
            set_pab_manager(config.pab_config)
        self._set_parallel()

    def _load_vae(self):
        """The native decoder of ``config.vae`` in the pipeline dtype (reference :214-215)."""
        v = self._config.vae
        if v is None:
            return None
        if not isinstance(v, AutoencoderKL):
            v = AutoencoderKL.from_pretrained(os.fspath(v), subfolder="vae")
        return v.to(self._dtype).to(self._device).eval()

    def decode_latents_to_video(self, latents, output_type: str = "pil"):
        """Reference :980-986 on latents [1, F, C, h, w]: ``[[frame_0, ...]]``, each frame post-processed on its own
        ("pil": a PIL image, "np": [H, W, 3] float32, "pt": [3, H, W]).  The frames are decoded several per pass: each
        is its own GroupNorm sample, so the result is the reference's frame-by-frame decode."""
        latents = (latents / self.vae.config.scaling_factor) + self.vae.config.shift_factor
        frames = decode_image_frames(self.vae, latents[0])
        return [list(postprocess_frames(frames, output_type))]

    def _embeds(self, prompt, negative_prompt, L=333):
        """Synthetic caption embeddings (77 CLIP + 256 T5 tokens, :498) when no text encoder is supplied."""
        cfg = self.transformer.config
        if self._config.text_encoder_fn is not None:
            return self._config.text_encoder_fn(prompt, negative_prompt)
        g = torch.Generator(device="cpu").manual_seed(zlib.crc32(str(prompt).encode()))
        mk = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
        return (mk(1, L, cfg.joint_attention_dim), mk(1, L, cfg.joint_attention_dim), mk(1, cfg.pooled_projection_dim),
                mk(1, cfg.pooled_projection_dim))

    @torch.no_grad()
    def generate(self, prompt=None, prompt_2=None, prompt_3=None, height: int = 288, width: int = 480, frames: int = 40,
                 num_inference_steps: int = 100, timesteps=None, guidance_scale: float = 7.5, seed: int = -1,
                 negative_prompt=None, negative_prompt_2=None, negative_prompt_3=None, num_images_per_prompt: int = 1,
                 generator=None, latents=None, prompt_embeds=None, negative_prompt_embeds=None, pooled_prompt_embeds=None,
                 negative_pooled_prompt_embeds=None, output_type: str = "pil", return_dict: bool = True,
                 joint_attention_kwargs=None, clip_skip=None, callback_on_step_end=None,
                 callback_on_step_end_tensor_inputs=("latents",)):
        if height % 8 or width % 8:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")  # :589-590
        update_steps(num_inference_steps)
        self.transformer.reset_pab_state()
        self._maybe_seed(seed)
        dev, dt = self._device, self._dtype
        if prompt_embeds is None:
            prompt_embeds, negative_prompt_embeds, pooled_prompt_embeds, negative_pooled_prompt_embeds = self._embeds(
                prompt, negative_prompt)
        do_cfg = guidance_scale > 1
        pe = [prompt_embeds.to(dev, dt)]
        pp = [pooled_prompt_embeds.to(dev, dt)]
        if do_cfg:
            pe.insert(0, negative_prompt_embeds.to(dev, dt))
            pp.insert(0, negative_pooled_prompt_embeds.to(dev, dt))
        self.scheduler.set_timesteps(num_inference_steps, dev)
        ts_host = [float(v) for v in self.scheduler.timesteps.tolist()]
        cin = self.transformer.config.in_channels
        if latents is None:
            latents = torch.randn(1, frames, cin, height // self.vae_scale_factor, width // self.vae_scale_factor, device=dev,
                                  dtype=dt)
        lat = latents.to(dev, dt)
        for i, t in enumerate(ts_host):
            tt = self.scheduler.timesteps[i].expand(1)
            ti = int(t) if enable_pab() else None  # the gates see int(timestep[0]) (attentions.py:839)
            preds = [self.transformer(lat, encoder_hidden_states=e, pooled_projections=p, timestep=tt, return_dict=False,
                                      ts_int=ti)[0] for e, p in zip(pe, pp)]
            if do_cfg:
                # :943-947.  As in the reference, the two forwards above share the attention modules' PAB counters and
                # caches (every gate advances twice per step)
                ramp = (1 - math.cos(math.pi * ((num_inference_steps - t) / num_inference_steps) ** 5.0)) / 2
                g = 1 + guidance_scale * ramp
                noise = preds[0] + g * (preds[1] - preds[0])
            else:
                noise = preds[0]
            lat = self.scheduler.step(noise, t, lat)[0]
        if self._config.vae_decode_fn is not None and output_type != "latents":
            video = self._config.vae_decode_fn(lat)
        elif self.vae is not None and output_type != "latents":
            video = self.decode_latents_to_video(lat, output_type)
        else:
            video = lat.float().cpu()  # latents
        return VideoSysPipelineOutput(video=video) if return_dict else (video,)
