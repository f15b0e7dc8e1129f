"""OpenSora pipeline surface (mirror of videosys/pipelines/open_sora/pipeline_open_sora.py: OpenSoraPABConfig :32-69,
OpenSoraConfig :126-163, OpenSoraPipeline.generate :426-656) around the native STDiT3.

In scope: the config classes, ``generate()``'s signature, the shape tables, the RFLOW loop and the denoiser, the VAE
decode on the native OpenSora v1.2 decoder (models/autoencoders/autoencoder_kl_open_sora.py), and the reference's
conditioning: image references (``refs``), mask strategies (``ms``) and looped generation (``loop``), on the native
encoder (conditioning.py).  Out of scope (SURVEY.md 2.1 row 7): the T5 text encoder, prompt cleaning and the aes / flow /
camera_motion score suffixes -- pass a ``text_encoder_fn``; without it ``generate`` feeds a deterministic synthetic
caption embedding.

The decode is opt-in: ``OpenSoraConfig(vae=<local snapshot directory or VideoAutoencoderPipeline instance>)`` makes
``generate`` return the reference's uint8 video ``[B, T, H, W, 3]`` (:638-648).  The default ``vae`` is the hub id
"hpcai-tech/OpenSora-VAE-v1.2", which is not a local directory, so by default ``generate`` returns the denoised LATENTS
exactly as before (the quantity the metric is defined on).  A ``vae_decode_fn`` takes precedence over both.  Under
sequence parallelism every rank decodes the whole video, and encodes its own references with the broadcast seed, as the
reference does.

Conditioning (``refs``, ``ms`` or ``loop > 1``) needs the native decoder and the native encoder
(``OpenSoraConfig(vae_encoder=<snapshot directory or OpenSoraVAEEncoder>)``, by default the ``vae`` directory), loaded on
the first ``generate`` that conditions; without them it raises ValueError.  It follows the reference's order (:519-643):
the prompt's JSON, every reference encoded, the loop prompts, then per loop the previous clip re-encoded and appended as a
reference (loop > 0), z drawn, the mask strategies applied, RFLOW with the mask, the decode.

Deliberate deviation: the reference trims and joins the loop clips along dim 1 of ``[B, C, T, H, W]`` (:641-643), the
channel axis, so ``[:, 17:]`` of 3 channels is empty and it returns only the first clip.  Here each later clip loses its
first ``dframe_to_frame(condition_frame_length)`` frames and the clips join along TIME (upstream Open-Sora's per-sample
``[:, dframe_to_frame(cfl):]`` on ``[C, T, H, W]``): ``nf + (loop - 1) * (nf - dframe_to_frame(cfl))`` frames.
"""
import zlib
from dataclasses import dataclass
from typing import Callable, Optional

import torch

from ...core.pab.pab_mgr import PABConfig, set_pab_manager, update_steps
from ...models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config
from ...schedulers.scheduling_rflow_open_sora import RFLOW
from . import conditioning as C

# 9:16 ("0.56") and 1:1 base sizes of pipelines/open_sora/data_process.py:63-235; other ratios are not tabulated here
_IMAGE_SIZE = {
    ("144p", "9:16"): (144, 256), ("240p", "9:16"): (240, 426), ("360p", "9:16"): (360, 640),
    ("480p", "9:16"): (480, 854), ("720p", "9:16"): (720, 1280), ("1080p", "9:16"): (1080, 1920),
    ("144p", "1:1"): (192, 192), ("240p", "1:1"): (320, 320), ("360p", "1:1"): (480, 480),
    ("480p", "1:1"): (640, 640), ("720p", "1:1"): (960, 960),
}
_NUM_FRAMES = {"1x": 51, "2x": 102, "4x": 204, "8x": 408, "16x": 816, "2s": 51, "4s": 102, "8s": 204, "16s": 408, "32s": 816}


def get_image_size(resolution: str, aspect_ratio: str):
    try:
        return _IMAGE_SIZE[(resolution, aspect_ratio)]
    except KeyError:
        raise ValueError(f"({resolution}, {aspect_ratio}) is not tabulated in videosys_b200 (9:16 and 1:1 only)") from None


def get_num_frames(num_frames):
    return _NUM_FRAMES[num_frames] if num_frames in _NUM_FRAMES else int(num_frames)


def get_latent_size(num_frames: int, height: int, width: int):
    """OpenSora VAE latent grid (models/autoencoders/autoencoder_kl_open_sora.py:706-717): 17-frame micro batches
    -> 5 latent frames each (time factor 4 with padding), 8x spatial."""
    t = (num_frames // 17) * 5
    rem = num_frames % 17
    if rem:
        t += -(-rem // 4)
    return t, height // 8, width // 8


class OpenSoraPABConfig(PABConfig):
    def __init__(self, spatial_broadcast=True, spatial_threshold=(450, 930), spatial_range=2, temporal_broadcast=True,
                 temporal_threshold=(450, 930), temporal_range=4, cross_broadcast=True, cross_threshold=(450, 930),
                 cross_range=6, mlp_broadcast=False, mlp_spatial_broadcast_config=None,
                 mlp_temporal_broadcast_config=None):
        # The reference defaults mlp_broadcast=True, which raises TypeError in STDiT3 at this commit because
        # all_timesteps never reaches the blocks (SURVEY.md fact 7); the only runnable setting is False.
        if mlp_broadcast:
            raise ValueError("mlp_broadcast is unreachable for OpenSora in the reference (SURVEY.md fact 7)")
        super().__init__(
            spatial_broadcast=spatial_broadcast, spatial_threshold=list(spatial_threshold), spatial_range=spatial_range,
            temporal_broadcast=temporal_broadcast, temporal_threshold=list(temporal_threshold),
            temporal_range=temporal_range, cross_broadcast=cross_broadcast, cross_threshold=list(cross_threshold),
            cross_range=cross_range, mlp_broadcast=False,
            mlp_spatial_broadcast_config=mlp_spatial_broadcast_config,
            mlp_temporal_broadcast_config=mlp_temporal_broadcast_config,
        )


class OpenSoraConfig:
    def __init__(self, transformer: str = "hpcai-tech/OpenSora-STDiT-v3", vae: str = "hpcai-tech/OpenSora-VAE-v1.2",
                 text_encoder: str = "DeepFloyd/t5-v1_1-xxl", num_gpus: int = 1, num_sampling_steps: int = 30,
                 cfg_scale: float = 7.0, cpu_offload: bool = False, tiling_size: int = 4,
                 enable_flash_attn: bool = False, enable_pab: bool = False, pab_config=None,
                 transformer_config: Optional[STDiT3Config] = None, state_dict=None,
                 text_encoder_fn: Optional[Callable] = None, vae_decode_fn: Optional[Callable] = None,
                 vae_encoder=None, fp8_linears: bool = False):
        self.pipeline_cls = OpenSoraPipeline
        # vae: a local snapshot directory of hpcai-tech/OpenSora-VAE-v1.2 or a VideoAutoencoderPipeline instance decodes
        # natively; anything else (the default hub id) leaves generate() returning latents
        self.transformer, self.vae, self.text_encoder = transformer, vae, text_encoder
        # vae_encoder: a local snapshot directory or an OpenSoraVAEEncoder instance for refs / ms / loop; None: the vae
        # directory when vae is one
        self.vae_encoder = vae_encoder
        self.num_gpus = num_gpus
        self.num_sampling_steps = num_sampling_steps
        self.cfg_scale = cfg_scale
        self.cpu_offload = cpu_offload
        self.tiling_size = tiling_size
        self.enable_flash_attn = enable_flash_attn
        self.enable_pab = enable_pab
        self.pab_config = pab_config if pab_config is not None else OpenSoraPABConfig()
        # native build extras: architecture / weights / out-of-scope stages supplied by the caller
        self.transformer_config = transformer_config
        self.state_dict = state_dict
        self.text_encoder_fn = text_encoder_fn
        self.vae_decode_fn = vae_decode_fn
        # FP8 mode of the denoiser (STDiT3.set_fp8_linears): the six block Linears on e4m3 operands; off keeps the bf16 path
        self.fp8_linears = fp8_linears


@dataclass
class VideoSysPipelineOutput:
    video: torch.Tensor


class OpenSoraPipeline:
    def __init__(self, config: OpenSoraConfig, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("videosys_b200 pipelines need an sm_90a GPU (no CPU path)")
        self._config = config
        self._device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        import os

        if config.transformer_config is None and config.state_dict is None and os.path.isdir(str(config.transformer)):
            # a local snapshot of hpcai-tech/OpenSora-STDiT-v3 (reference :222-224 downloads it)
            self.transformer = STDiT3.from_pretrained(config.transformer, enable_flash_attn=config.enable_flash_attn).to(torch.bfloat16)
        else:
            tcfg = config.transformer_config or STDiT3Config(depth=28, hidden_size=1152, num_heads=16)
            self.transformer = STDiT3(tcfg).to(torch.bfloat16)
        if config.state_dict is not None:
            self.transformer.load_state_dict(config.state_dict)
        self.transformer = self.transformer.to(self._device).eval()
        if config.fp8_linears:
            self.transformer.set_fp8_linears(True)
        self.scheduler = RFLOW(num_sampling_steps=config.num_sampling_steps, cfg_scale=config.cfg_scale,
                               use_timestep_transform=True)
        self.vae = self._load_vae()
        self._vae_encoder = None  # loaded by the first generate that conditions
        if config.enable_pab:
            set_pab_manager(config.pab_config)
        self._set_parallel()

    def _load_vae(self):
        """The native VAE of ``config.vae`` in bf16 on the pipeline's device (the reference builds it with
        micro_batch_size = config.tiling_size, :215-220), or None when ``config.vae`` is not a local directory or an
        instance."""
        from ...models.autoencoders.autoencoder_kl_open_sora import load_vae

        vae = load_vae(self._config.vae, micro_batch_size=self._config.tiling_size)
        return None if vae is None else vae.to(torch.bfloat16).to(self._device).eval()

    def _load_vae_encoder(self):
        """The native encoder for conditioning, in bf16 on the pipeline's device (loaded once), or None."""
        if self._vae_encoder is None:
            from ...models.autoencoders.autoencoder_kl_open_sora import load_vae_encoder

            enc = load_vae_encoder(self._config.vae_encoder, self._config.vae, micro_batch_size=self._config.tiling_size)
            self._vae_encoder = None if enc is None else enc.to(torch.bfloat16).to(self._device).eval()
        return self._vae_encoder

    def decode_latents(self, samples, num_frames: int):
        """The reference tail (:638-648): vae(samples, decode_only=True, num_frames), then clamp_(-1, 1), sub_(-1),
        div_(2), mul(255), add_(0.5), clamp_(0, 255) in bf16, as uint8 [B, T, H, W, 3] on the CPU."""
        return self._to_uint8(self.vae.decode(samples.to(torch.bfloat16), num_frames=num_frames))

    @staticmethod
    def _to_uint8(video):
        low, high = -1, 1
        video.clamp_(min=low, max=high)
        video.sub_(low).div_(max(high - low, 1e-5))
        return video.mul(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 4, 1).to("cpu", torch.uint8)

    def _check_conditioning(self, loop, condition_frame_length):
        """refs / ms / loop need the native decoder and encoder (the decoded clips are re-encoded); raises ValueError."""
        if loop < 1:
            raise ValueError(f"loop={loop} must be >= 1")
        if self._config.vae_decode_fn is not None:
            raise ValueError("refs / ms / loop decode and re-encode on the native VAE: do not pass vae_decode_fn")
        if getattr(self, "vae", None) is None or self._load_vae_encoder() is None:
            raise ValueError("refs / ms / loop need the native OpenSora v1.2 VAE: OpenSoraConfig(vae=<local snapshot "
                             "directory or VideoAutoencoderPipeline>, vae_encoder=<directory or OpenSoraVAEEncoder>)")
        if loop > 1:
            C.dframe_to_frame(condition_frame_length)

    def _set_parallel(self, dp_size=None, sp_size=None, enable_cp=False):
        import torch.distributed as dist

        world = dist.get_world_size() if dist.is_initialized() else 1
        if sp_size is None:
            sp_size, dp_size = world, 1
        else:
            dp_size = world // sp_size
        self.transformer.enable_parallel(dp_size, sp_size, enable_cp)

    def _set_seed(self, seed: int):
        """Reference set_seed (utils/utils.py:19-34): seed == -1 draws one, rank 0's value is BROADCAST so that every rank
        of a sequence-parallel group denoises the same latent (each rank draws z and the per-step noise itself), the dp
        rank is added, then python / numpy / torch generators are seeded."""
        import random

        import numpy as np
        import torch.distributed as dist

        if seed is None or seed == -1:
            seed = random.randint(0, 1000000)
        if dist.is_initialized() and dist.get_world_size() > 1:
            t = torch.tensor([seed], dtype=torch.int64, device=self._device)
            dist.broadcast(t, src=0)
            seed = int(t.item())
        pm = self.transformer.parallel_manager
        seed = int(seed) + (pm.dp_rank if pm is not None else 0)
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        torch.cuda.manual_seed(seed)
        return seed

    def _encode_text(self, prompt: str, negative: str = ""):
        cfg = self.transformer.config
        if self._config.text_encoder_fn is not None:
            return self._config.text_encoder_fn(prompt, negative)
        g = torch.Generator(device="cpu").manual_seed(zlib.crc32(prompt.encode()))
        y = torch.randn(1, 1, cfg.model_max_length, cfg.caption_channels, generator=g)
        mask = torch.ones(1, cfg.model_max_length, dtype=torch.long)
        y_null = self.transformer.y_embedder.y_embedding[None, None].float().cpu()
        return y, mask, y_null

    @torch.no_grad()
    def generate(self, prompt, resolution="480p", aspect_ratio="9:16", num_frames: int = 51, loop: int = 1,
                 llm_refine: bool = False, negative_prompt: str = "", seed: int = -1, ms: Optional[str] = "",
                 refs: Optional[str] = "", aes: float = 6.5, flow: Optional[float] = None,
                 camera_motion: Optional[float] = None, condition_frame_length: int = 5, align: int = 5,
                 condition_frame_edit: float = 0.0, return_dict: bool = True, verbose: bool = True):
        prompts, refs_l, ms_l = C.extract_json_from_prompts([prompt], [refs or ""], [ms or ""])
        conditioned = loop != 1 or bool(refs_l[0]) or bool(ms_l[0])
        if conditioned:
            self._check_conditioning(loop, condition_frame_length)
        dev, dtype = self._device, torch.bfloat16
        image_size = get_image_size(resolution, aspect_ratio)
        nf = get_num_frames(num_frames)
        fps = 24 if nf > 1 else 120  # IMG_FPS for single images (reference prepare_multi_resolution_info)
        Tl_chk = get_latent_size(nf, *image_size)[0]
        if Tl_chk == 1 and self.transformer.parallel_manager is not None and self.transformer.parallel_manager.sp_size > 1:
            raise NotImplementedError("single-image generation under sequence parallelism (the reference scatters the "
                                      "batch for images, open_sora_transformer_3d.py:292-296): use num_gpus=1")
        update_steps(self._config.num_sampling_steps)
        self.transformer.reset_pab_state()
        self._set_seed(seed)
        encode = None
        refs_x = [[]]
        if conditioned:  # every reference encoded now, before z, as the reference does (:532-535)
            enc = self._vae_encoder
            encode = lambda x: enc.encode(x.to(enc.device, enc.dtype))  # noqa: E731
            refs_x = C.collect_references_batch(refs_l, encode, image_size)
        texts, loop_idx = C.split_prompt(prompts[0])
        batch_prompts = [C.merge_prompt(texts, loop_idx)]
        Tl, Hl, Wl = get_latent_size(nf, *image_size)
        clips = []
        for loop_i in range(loop):
            prompt_i = C.extract_prompts_loop(batch_prompts, loop_i)[0]
            if loop_i > 0:  # the previous clip re-encoded as the next one's first frames (:614-617)
                refs_x, ms_l = C.append_generated(encode, clips[-1], refs_x, ms_l, loop_i, condition_frame_length,
                                                  condition_frame_edit)
            y, mask, y_null = self._encode_text(prompt_i, negative_prompt)  # before z, as without conditioning
            z = torch.randn(1, self.transformer.in_channels, Tl, Hl, Wl, device=dev, dtype=dtype)
            margs = dict(
                y=y.to(dev, dtype), mask=mask.to(dev),
                height=torch.tensor([image_size[0]], device=dev, dtype=dtype),
                width=torch.tensor([image_size[1]], device=dev, dtype=dtype),
                num_frames=torch.tensor([nf], device=dev, dtype=dtype),
                fps=torch.tensor([fps], device=dev, dtype=dtype),
            )
            # ms = "" gives an all-ones mask (:825-854)
            masks = C.apply_mask_strategy(z, refs_x, ms_l, loop_i, align=align)
            samples = self.scheduler.sample(self.transformer, z, margs, y_null.to(dev, dtype), dev, mask=masks,
                                            progress=verbose)
            if conditioned:
                clips.append(self.vae.decode(samples.to(dtype), num_frames=nf))
        if conditioned:
            # the loop clips join along TIME, each later one without its conditioning frames (module docstring)
            cut = C.dframe_to_frame(condition_frame_length) if loop > 1 else 0
            video = self._to_uint8(torch.cat([clips[0]] + [c[:, :, cut:] for c in clips[1:]], dim=2))
        elif self._config.vae_decode_fn is not None:
            video = self._config.vae_decode_fn(samples, nf)
        elif getattr(self, "vae", None) is not None:
            video = self.decode_latents(samples, nf)
        else:
            video = samples.float().cpu()  # latents: no local VAE
        return VideoSysPipelineOutput(video=video) if return_dict else (video,)
