"""Writes tests/golden/latte_vae.pt and tests/golden/vchitect_vae.pt: the decode tails of the reference Latte and
Vchitect-2.0 pipelines on the restated diffusers VAEs (oracle/svd_vae_ref.py, oracle/sd_vae_ref.py) in fp32 on the CPU.

    python -m oracle.gen_golden_latte_vae

The reference's pipeline modules import diffusers at load time, so their decode tails are restated below with line
citations.  Only outputs are stored: a seeded random subset of ``SAMPLES`` elements (``sample_index``) and the shape, of
the float video before the pipelines' final conversions (Latte's uint8 cast, Vchitect's ``VaeImageProcessor``).  Weights
and latents are regenerated from seeds (``weights`` of gen_golden_opensora_vae, ``latents``).
"""
import os
import types
import zlib

import torch
import torch.nn as nn

from oracle.gen_golden_opensora_vae import NARROW, RELEASED, weights

SAMPLES = 8000
VCH_SCALE, VCH_SHIFT = 1.5305, 0.0609  # Vchitect-2.0's vae/config.json (the SD3 VAE)
# name -> (decoder, widths, latent shape).  Latte latents are [B, 4, F, h, w], Vchitect's [1, F, 16, h, w]
LATTE_CASES = {
    "temporal_16": ("temporal", NARROW, (1, 4, 16, 2, 3)),  # chunks of 14 + 2 frames
    "temporal_b2": ("temporal", NARROW, (2, 4, 16, 2, 2)),  # chunks of 14, 14, 4: the middle one straddles the samples
    "image": ("sd", NARROW, (1, 4, 1, 3, 2)),               # video_length 1: decode_latents_image
    "sd_vae": ("sd", NARROW, (1, 4, 3, 2, 3)),              # enable_vae_temporal_decoder=False
    "temporal_released": ("temporal", RELEASED, (1, 4, 2, 2, 2)),
}
VCHITECT_CASES = {
    "narrow": (NARROW, (1, 3, 16, 2, 3)),
    "released": (RELEASED, (1, 2, 16, 2, 2)),
}


class VchitectVAE(nn.Module):
    """diffusers' AutoencoderKL with latent_channels 16 and use_post_quant_conv False (oracle/sd_vae_ref.py's decoder)."""

    def __init__(self, block_out_channels):
        super().__init__()
        from oracle.sd_vae_ref import Decoder

        self.config = types.SimpleNamespace(scaling_factor=VCH_SCALE, shift_factor=VCH_SHIFT, latent_channels=16)
        self.decoder = Decoder(16, block_out_channels, 2)

    def decode(self, z, return_dict=True):
        s = self.decoder(z)
        return types.SimpleNamespace(sample=s) if return_dict else (s,)


def build_latte_vae(kind, widths):
    if kind == "temporal":
        from oracle.svd_vae_ref import AutoencoderKLTemporalDecoder

        return AutoencoderKLTemporalDecoder(widths)
    from oracle.sd_vae_ref import AutoencoderKL

    vae = AutoencoderKL(widths)
    vae.config.scaling_factor = 0.18215
    return vae


# ---- the reference's decode tails (videosys/pipelines/latte/pipeline_latte.py, pipelines/vchitect/pipeline_vchitect.py)
def _frames(latents):  # einops "b c f h w -> (b f) c h w"
    b, c, f, h, w = latents.shape
    return latents.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)


def latte_decode_image(vae, latents):
    """pipeline_latte.py:904-914: float [b, f, c, h, w] in [0, 1]."""
    b, _, f = latents.shape[:3]
    latents = _frames(1 / vae.config.scaling_factor * latents)
    video = torch.cat([vae.decode(latents[i:i + 1]).sample for i in range(latents.shape[0])])
    return (video.reshape(b, f, *video.shape[1:]) / 2.0 + 0.5).clamp(0, 1)


def latte_decode_video(vae, latents, temporal):
    """pipeline_latte.py:916-925 (per frame) or :927-946 (chunks of 14 frames, num_frames = the chunk's length), up to
    the uint8 cast: float [b, f, h, w, c]."""
    b, _, f = latents.shape[:3]
    latents = _frames(1 / vae.config.scaling_factor * latents)
    if temporal:
        video = [vae.decode(latents[i:i + 14], num_frames=latents[i:i + 14].shape[0]).sample
                 for i in range(0, latents.shape[0], 14)]
    else:
        video = [vae.decode(latents[i:i + 1]).sample for i in range(latents.shape[0])]
    video = torch.cat(video)
    return video.reshape(b, f, *video.shape[1:]).permute(0, 1, 3, 4, 2)


def latte_to_uint8(video):
    """pipeline_latte.py:923-924 / :944-945."""
    return ((video / 2.0 + 0.5).clamp(0, 1) * 255).to(dtype=torch.uint8).cpu().contiguous()


def vchitect_decode(vae, latents):
    """pipeline_vchitect.py:980-984 up to the post-processing: the decoded frames [F, 3, H, W] of sample 0."""
    latents = (latents / vae.config.scaling_factor) + vae.config.shift_factor
    return torch.cat([vae.decode(latents[:, v], return_dict=False)[0][:1] for v in range(latents.shape[1])])


def latents(name, shape, dtype=torch.float32):
    g = torch.Generator().manual_seed(zlib.crc32(f"latents/{name}".encode()))
    return torch.randn(shape, generator=g).to(dtype)


def sample_index(numel, name):
    g = torch.Generator().manual_seed(zlib.crc32(f"sample/{name}".encode()))
    return torch.randperm(numel, generator=g)[:SAMPLES]


def latte_case(name):
    """(reference vae with the case's weights, latents, float output) of a Latte case."""
    kind, widths, shape = LATTE_CASES[name]
    vae = build_latte_vae(kind, widths)
    vae.load_state_dict(weights(vae.state_dict(), "latte/" + name))
    z = latents("latte/" + name, shape)
    if shape[2] == 1:
        return vae, z, latte_decode_image(vae, z)
    return vae, z, latte_decode_video(vae, z, kind == "temporal")


def vchitect_case(name):
    widths, shape = VCHITECT_CASES[name]
    vae = VchitectVAE(widths)
    vae.load_state_dict(weights(vae.state_dict(), "vchitect/" + name))
    z = latents("vchitect/" + name, shape)
    return vae, z, vchitect_decode(vae, z)


def _store(out, name, y):
    out[f"{name}.shape"] = list(y.shape)
    flat = y.flatten()
    out[f"{name}.fp32"] = flat[sample_index(flat.numel(), name)].clone() if flat.numel() > SAMPLES else flat.clone()
    print(name, tuple(y.shape), float(y.abs().mean()))


def main():
    torch.set_grad_enabled(False)
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
    for fname, cases, run in (("latte_vae.pt", LATTE_CASES, latte_case), ("vchitect_vae.pt", VCHITECT_CASES, vchitect_case)):
        out = {}
        for name in cases:
            _store(out, name, run(name)[2])
        path = os.path.join(root, fname)
        torch.save(out, path)
        print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
