"""CogVideoX pipeline surface (mirror of videosys/pipelines/cogvideox/pipeline_cogvideox.py: CogVideoXPABConfig :33-44,
CogVideoXConfig :47-112, CogVideoXPipeline.generate :489-737) around the native CogVideoXTransformer3DModel.

In scope: the config classes, ``generate()``'s signature and shape rules, the CFG + DDIM denoising loop (:692-733),
the denoiser, and -- opt-in through ``CogVideoXConfig(vae=...)`` -- the VAE decode tail (:359-364, :739-741) on the native
decoder (models/autoencoders/autoencoder_kl_cogvideox.py).  Out of scope as for OpenSora (SURVEY.md 2.1): the T5 encoder
-- pass ``prompt_embeds`` / ``negative_prompt_embeds`` or a ``text_encoder_fn``.  Without a ``vae`` or a ``vae_decode_fn``
the LATENTS are returned (``output_type="latent"`` semantics).  dtype follows the reference: fp16 for
"THUDM/CogVideoX-2b", else bf16.

The video post-processing restates diffusers' ``VideoProcessor.postprocess_video`` (pipelines/_common.py, diffusers is not
a dependency): ``(x / 2 + 0.5).clamp(0, 1)`` per frame, then "pt" -> [B, F, 3, H, W], "np" -> [B, F, H, W, 3], "pil" ->
lists of PIL images.
"""
import zlib
from typing import Callable, Optional

import torch

from ...core.pab.pab_mgr import PABConfig, enable_pab, set_pab_manager, update_steps
from ...models.transformers.cogvideox_transformer_3d import CogVideoXTransformer3DModel
from ...schedulers.scheduling_ddim_cogvideox import CogVideoXDDIMScheduler
from .._common import ParallelPipelineMixin, postprocess_frames
from ..open_sora.pipeline_open_sora import VideoSysPipelineOutput


class CogVideoXPABConfig(PABConfig):
    def __init__(self, spatial_broadcast: bool = True, spatial_threshold: list = (100, 850), spatial_range: int = 2):
        super().__init__(spatial_broadcast=spatial_broadcast, spatial_threshold=list(spatial_threshold), spatial_range=spatial_range)


class CogVideoXConfig:
    def __init__(self, model_path: str = "THUDM/CogVideoX-2b", num_gpus: int = 1, cpu_offload: bool = False,
                 vae_tiling: bool = True, enable_pab: bool = False, pab_config=None,
                 transformer_config: Optional[dict] = None, state_dict=None, text_encoder_fn: Optional[Callable] = None,
                 vae_decode_fn: Optional[Callable] = None, vae=None):
        self.model_path = model_path
        self.pipeline_cls = CogVideoXPipeline
        self.num_gpus = num_gpus
        self.cpu_offload = cpu_offload
        self.vae_tiling = vae_tiling
        self.enable_pab = enable_pab
        self.pab_config = pab_config if pab_config is not None else CogVideoXPABConfig()
        # native build extras (as OpenSoraConfig): architecture / weights / out-of-scope stages supplied by the caller
        self.transformer_config = transformer_config
        self.state_dict = state_dict
        self.text_encoder_fn = text_encoder_fn
        self.vae_decode_fn = vae_decode_fn
        # native VAE decoder: a local snapshot directory (its root or its vae/ folder) or an AutoencoderKLCogVideoX
        self.vae = vae


class CogVideoXPipeline(ParallelPipelineMixin):
    vae_scale_factor_spatial = 8
    vae_scale_factor_temporal = 4

    def __init__(self, config: CogVideoXConfig, device=None, dtype: torch.dtype = torch.bfloat16):
        if not torch.cuda.is_available():
            raise RuntimeError("videosys_b200 pipelines need an sm_90a GPU (no CPU path)")
        self._config = config
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if config.model_path == "THUDM/CogVideoX-2b":
            dtype = torch.float16  # reference :138-139
        self._dtype = dtype
        import os

        if config.transformer_config is None and config.state_dict is None and os.path.isdir(str(config.model_path)):
            self.transformer = CogVideoXTransformer3DModel.from_pretrained(config.model_path, subfolder="transformer").to(dtype)
        else:
            tc = config.transformer_config
            if tc is None and "5b" in str(config.model_path).lower():  # THUDM/CogVideoX-5b: 48 heads x 64, 42 blocks, rotary
                tc = dict(num_attention_heads=48, num_layers=42, use_rotary_positional_embeddings=True)
            self.transformer = CogVideoXTransformer3DModel(**(tc or {})).to(dtype)
        if config.state_dict is not None:
            self.transformer.load_state_dict(config.state_dict)
        self.transformer = self.transformer.to(self._device).eval()
        self.scheduler = CogVideoXDDIMScheduler()
        self.vae = self._load_vae()
        if config.enable_pab:
            set_pab_manager(config.pab_config)
        self._set_parallel()

    def _load_vae(self):
        """The native decoder of ``config.vae`` in the pipeline dtype, with tiling as the reference sets it (:170-172)."""
        import os

        from ...models.autoencoders.autoencoder_kl_cogvideox import AutoencoderKLCogVideoX

        v = self._config.vae
        if v is None:
            return None
        if not isinstance(v, AutoencoderKLCogVideoX):
            v = str(v)
            v = AutoencoderKLCogVideoX.from_pretrained(v, subfolder="vae" if os.path.isdir(os.path.join(v, "vae")) else "")
        v = v.to(self._dtype).to(self._device).eval()
        if self._config.vae_tiling:
            v.enable_tiling()
        return v

    def decode_latents_to_video(self, latents, output_type: str = "pil"):
        """Reference decode_latents (:359-364) and VideoProcessor.postprocess_video: latents [B, F, C, h, w]."""
        z = latents.permute(0, 2, 1, 3, 4)
        z = 1 / self.vae.config.scaling_factor * z
        frames = self.vae.decode(z).sample  # [B, 3, F, H, W]
        return postprocess_frames(frames.permute(0, 2, 1, 3, 4), output_type)

    def _embeds(self, prompt, negative_prompt, max_sequence_length):
        cfg = self.transformer.config
        if self._config.text_encoder_fn is not None:
            return self._config.text_encoder_fn(prompt, negative_prompt)
        g = torch.Generator(device="cpu").manual_seed(zlib.crc32(str(prompt).encode()))
        pe = torch.randn(1, max_sequence_length, cfg.text_embed_dim, generator=g)
        ne = torch.randn(1, max_sequence_length, cfg.text_embed_dim, generator=g)
        return pe, ne

    def prepare_latents(self, batch, channels, num_frames, height, width, dtype, device, latents=None):
        shape = (batch, (num_frames - 1) // self.vae_scale_factor_temporal + 1, channels,
                 height // self.vae_scale_factor_spatial, width // self.vae_scale_factor_spatial)
        if latents is None:
            latents = torch.randn(shape, device=device, dtype=dtype)
        return latents.to(device) * self.scheduler.init_noise_sigma

    def _prepare_rotary_positional_embeddings(self, height: int, width: int, num_frames: int, device):
        """Reference :449-474 (get_resize_crop_region_for_grid :758-773, get_3d_rotary_pos_embed models/modules/
        embeddings.py:283-364): (cos, sin) [frames * grid_h * grid_w, head_dim] fp32 of the video tokens."""
        import numpy as np

        cfg = self.transformer.config
        unit = self.vae_scale_factor_spatial * cfg.patch_size
        gh, gw = height // unit, width // unit
        tw, th = 720 // unit, 480 // unit
        if gh / gw > th / tw:
            rh, rw = th, int(round(th / gh * gw))
        else:
            rw, rh = tw, int(round(tw / gw * gh))
        top, left = int(round((th - rh) / 2.0)), int(round((tw - rw) / 2.0))
        D, theta = cfg.attention_head_dim, 10000.0
        lin = lambda a, b, n: torch.from_numpy(np.linspace(a, b, n, endpoint=False, dtype=np.float32)).float()  # noqa: E731

        def freqs(grid, d):
            f = 1.0 / (theta ** (torch.arange(0, d, 2).float() / d))
            return torch.einsum("n,f->nf", grid, f).repeat_interleave(2, dim=-1)

        ft = freqs(lin(0, num_frames, num_frames), D // 4)
        fh = freqs(lin(top, top + rh, gh), D // 8 * 3)
        fw = freqs(lin(left, left + rw, gw), D // 8 * 3)
        fr = torch.cat([ft[:, None, None, :].expand(num_frames, gh, gw, -1), fh[None, :, None, :].expand(num_frames, gh, gw, -1),
                        fw[None, None, :, :].expand(num_frames, gh, gw, -1)], dim=-1).reshape(num_frames * gh * gw, -1)
        return fr.cos().to(device), fr.sin().to(device)

    @torch.no_grad()
    def generate(self, prompt=None, negative_prompt=None, height: int = 480, width: int = 720, num_frames: int = 49,
                 num_inference_steps: int = 50, timesteps=None, seed: int = -1, guidance_scale: float = 6,
                 use_dynamic_cfg: bool = False, num_videos_per_prompt: int = 1, eta: float = 0.0, generator=None,
                 latents=None, prompt_embeds=None, negative_prompt_embeds=None, output_type: str = "pil",
                 return_dict: bool = True, callback_on_step_end=None, callback_on_step_end_tensor_inputs=("latents",),
                 max_sequence_length: int = 226):
        import math

        if num_frames > 49:
            raise ValueError("The number of frames must be less than 49 for now due to static positional embeddings.")
        if height % 8 or width % 8:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        update_steps(num_inference_steps)
        self.transformer.reset_pab_state()
        self._maybe_seed(seed)
        dev, dt = self._device, self._dtype
        if prompt_embeds is None:
            prompt_embeds, negative_prompt_embeds = self._embeds(prompt, negative_prompt, max_sequence_length)
        do_cfg = guidance_scale > 1.0
        pe = prompt_embeds.to(dev, dt)
        if do_cfg:
            pe = torch.cat([negative_prompt_embeds.to(dev, dt), pe], dim=0)  # reference order: [uncond, cond] (:646)
        self.scheduler.set_timesteps(num_inference_steps, dev)
        ts = self.scheduler.timesteps if timesteps is None else torch.as_tensor(timesteps, device=dev)
        ts_host = [int(v) for v in ts.tolist()]
        lat = self.prepare_latents(prompt_embeds.shape[0], self.transformer.config.in_channels, num_frames, height, width,
                                   dt, dev, latents)
        rotary = None
        if self.transformer.config.use_rotary_positional_embeddings:  # CogVideoX-5b (reference :669-673)
            rotary = self._prepare_rotary_positional_embeddings(height, width, lat.size(1), dev)
        gs = guidance_scale
        for i, t in enumerate(ts_host):
            inp = torch.cat([lat] * 2) if do_cfg else lat
            tt = torch.full((inp.shape[0],), t, device=dev, dtype=torch.int64)
            noise = self.transformer(hidden_states=inp, encoder_hidden_states=pe, timestep=tt, image_rotary_emb=rotary,
                                     return_dict=False, ts_int=t if enable_pab() else None)[0].float()
            if use_dynamic_cfg:
                gs = 1 + guidance_scale * ((1 - math.cos(math.pi * ((num_inference_steps - t) / num_inference_steps) ** 5.0)) / 2)
            if do_cfg:
                un, tx = noise.chunk(2)
                noise = un + gs * (tx - un)
            lat = self.scheduler.step(noise, t, lat, eta=eta)[0].to(dt)
        if self._config.vae_decode_fn is not None and output_type != "latent":
            video = self._config.vae_decode_fn(lat)
        elif self.vae is not None and output_type != "latent":
            video = self.decode_latents_to_video(lat, output_type)
        else:
            video = lat.float().cpu()  # latents: the VAE is out of scope
        return VideoSysPipelineOutput(video=video) if return_dict else (video,)
