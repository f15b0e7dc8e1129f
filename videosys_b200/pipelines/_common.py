"""What the CogVideoX and Latte pipelines share with the reference's: the process-mesh set-up (reference
pipeline_cogvideox.py:195-209 = pipeline_latte.py:261-275) and the seeding rule (utils/utils.py:19-34); and what the
pipelines that decode with an image VAE share: diffusers' video / image post-processing restated (diffusers is not a
dependency) and the frame batching of the image decoders."""
import random
from typing import Optional

import torch
import torch.distributed as dist


# image-VAE frames decoded per pass.  Each frame is its own GroupNorm sample, so the result does not depend on it; it
# bounds the activation memory (8 frames of 512 x 512 x 128 channels: 0.5 GB per 16-bit tensor)
VAE_FRAMES_PER_PASS = 8


def decode_image_frames(vae, z, **kwargs):
    """``vae.decode(z[i:i + n], **kwargs).sample`` over the frames of z [N, C, h, w], n = VAE_FRAMES_PER_PASS at a time
    -> [N, 3, 8h, 8w]."""
    n = VAE_FRAMES_PER_PASS
    return torch.cat([vae.decode(z[i:i + n], **kwargs).sample for i in range(0, z.shape[0], n)])


def postprocess_frames(frames, output_type: str = "pil"):
    """diffusers' ``VaeImageProcessor.postprocess`` / ``VideoProcessor.postprocess_video`` of decoded frames
    [..., 3, H, W] in [-1, 1]: ``(x / 2 + 0.5).clamp(0, 1)``, then "pt" -> the tensor [..., 3, H, W], "np" -> a float32
    array [..., H, W, 3], "pil" -> nested lists (one level per leading dimension) of PIL images."""
    video = (frames / 2 + 0.5).clamp(0, 1)
    if output_type == "pt":
        return video
    arr = video.movedim(-3, -1).float().cpu().numpy()
    if output_type == "np":
        return arr
    if output_type == "pil":
        from PIL import Image

        def pil(a):
            return Image.fromarray((a * 255).round().astype("uint8")) if a.ndim == 3 else [pil(f) for f in a]

        return pil(arr)
    raise ValueError(f"output_type={output_type!r}: expected 'pil', 'np', 'pt' or 'latent'")


class ParallelPipelineMixin:
    """Needs ``self.transformer`` (with ``enable_parallel`` / ``parallel_manager``) and ``self._device``."""

    def _set_parallel(self, dp_size: Optional[int] = None, sp_size: Optional[int] = None, enable_cp: Optional[bool] = False):
        """Every rank joins one sequence-parallel group unless told otherwise; ``enable_cp`` turns a factor 2 of it into
        CFG parallelism (the transformer's ``enable_parallel``)."""
        world = dist.get_world_size() if dist.is_initialized() else 1
        if sp_size is None:
            sp_size, dp_size = world, 1
        else:
            assert world % sp_size == 0, f"world_size {world} must be divisible by sp_size"
            dp_size = world // sp_size
        self.transformer.enable_parallel(dp_size, sp_size, enable_cp)

    def _set_seed(self, seed):
        """One seed per dp replica.  seed < 0 draws one; rank 0's draw is broadcast so that the ranks of a sequence- /
        CFG-parallel group denoise the same latent (every rank draws the latent itself)."""
        if seed is None or seed < 0:
            seed = random.randint(0, 1000000)
        if dist.is_initialized() and dist.get_world_size() > 1:
            t = torch.tensor([seed], dtype=torch.int64, device=self._device)
            dist.broadcast(t, src=0)
            seed = int(t.item())
        pm = self.transformer.parallel_manager
        seed = int(seed) + (pm.dp_rank if pm is not None else 0)
        random.seed(seed)
        torch.manual_seed(seed)
        torch.cuda.manual_seed(seed)
        return seed

    def _maybe_seed(self, seed):
        """Seed when asked to, and always under multi-GPU (unseeded ranks would draw different latents)."""
        if (seed is not None and seed >= 0) or (dist.is_initialized() and dist.get_world_size() > 1):
            self._set_seed(seed)
