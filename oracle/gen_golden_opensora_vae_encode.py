"""Writes tests/golden/opensora_vae_encode.pt: outputs of the UNMODIFIED reference OpenSora v1.2 VAE encode
(``VideoAutoencoderPipeline.encode`` with its image micro-batches and 17-frame chunks, ``VAE_Temporal.encode`` and its
``Encoder``, loaded by oracle/opensora_vae_ref.py; the SDXL AutoencoderKL encoder restated in oracle/sd_vae_encoder_ref.py)
in fp32 on the CPU.

    python -m oracle.gen_golden_opensora_vae_encode

Per case: ``z`` = (sample - shift) / scale with torch.manual_seed(SEED) set before ``encode`` (the CPU generator supplies
every Gaussian draw there), and ``mode`` = the same with the posteriors' means (the noise replaced by zeros), each as a
seeded subset of at most ``SAMPLES`` elements (``sample_index``) plus the shape.  Weights (``weights`` of the decode
golden, seeded by case and key) and videos (``videos``) are regenerated from seeds.
"""
import os

import torch

from oracle.gen_golden_opensora_vae import NARROW, RELEASED, weights

# name -> (spatial block_out_channels, video shape [B, 3, T, H, W])
# (latents of a few hundred elements or more, so that a norm over them is a stable statistic)
CASES = {
    "image": (NARROW, (1, 3, 1, 64, 104)),         # one frame: 3 zero padding frames in front
    "one_chunk": (NARROW, (1, 3, 17, 48, 64)),
    "remainder": (NARROW, (1, 3, 20, 48, 64)),     # 17 + a 3-frame chunk with 1 padding frame
    "batch2": (NARROW, (2, 3, 5, 48, 48)),
    "odd_width": (NARROW, (1, 3, 2, 64, 424)),     # a 240p-like width, 424 -> 212 -> 106 -> 53: the far-side pad matters
    "released": (RELEASED, (1, 3, 4, 48, 64)),
}
SEED = 1234
SAMPLES = 4000


def videos(name, dtype=torch.float32):
    """A seeded video in [-1, 1]."""
    g = torch.Generator().manual_seed(6100 + list(CASES).index(name))
    return (2 * torch.rand(CASES[name][1], generator=g) - 1).to(dtype)


def sample_index(numel, name):
    g = torch.Generator().manual_seed(7100 + list(CASES).index(name))
    return torch.randperm(numel, generator=g)[:SAMPLES]


def _subset(y, name):
    flat = y.flatten()
    return flat[sample_index(flat.numel(), name)].clone() if flat.numel() > SAMPLES else flat.clone()


def main():
    from oracle.sd_vae_encoder_ref import build_opensora_vae_full

    torch.set_grad_enabled(False)
    out = {}
    for name, (spatial, _) in CASES.items():
        ref = build_opensora_vae_full(spatial)
        ref.load_state_dict(weights(ref.state_dict(), name))
        torch.manual_seed(SEED)
        z = ref.encode(videos(name))
        with torch.random.fork_rng():
            torch.randn = _zeros_like_randn(torch.randn)
            try:
                mode = ref.encode(videos(name))
            finally:
                torch.randn = torch.randn.__wrapped__
        out[f"{name}.shape"] = list(z.shape)
        out[f"{name}.z"] = _subset(z, name)
        out[f"{name}.mode"] = _subset(mode, name)
        print(name, tuple(z.shape), float(z.abs().mean()), float(mode.abs().mean()))
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "opensora_vae_encode.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


def _zeros_like_randn(randn):
    """torch.randn replaced by zeros of the same shape / device / dtype: the posterior's sample becomes its mean."""
    def zeros(*shape, **kw):
        kw.pop("generator", None)
        return torch.zeros(*shape, **kw)
    zeros.__wrapped__ = randn
    return zeros


if __name__ == "__main__":
    main()
