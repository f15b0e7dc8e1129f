"""Writes tests/golden/opensora_vae.pt: outputs of the UNMODIFIED reference OpenSora v1.2 VAE decode
(oracle/opensora_vae_ref.py: ``VideoAutoencoderPipeline.decode`` with its micro-batching, scale / shift, temporal VAE and
``VideoAutoencoderKL.decode``; the SDXL AutoencoderKL body restated in oracle/sd_vae_ref.py) in fp32 on the CPU.

    python -m oracle.gen_golden_opensora_vae

Only outputs are stored: a seeded random subset of ``SAMPLES`` elements (``sample_index``) and the shape.  Weights and
latents are regenerated from seeds (``weights`` / ``latents``); each tensor is seeded by the case and its key, so the
reference's full state dict and the decoder-only one get the same values.  The temporal decoder always has its released
widths; the image decoder is narrow or released per case.
"""
import os
import zlib

import torch

NARROW = (64, 64, 128, 128)
RELEASED = (128, 256, 512, 512)
# name -> (spatial block_out_channels, latent shape [B, 4, T, h, w], num_frames)
CASES = {
    "one_chunk": (NARROW, (1, 4, 5, 4, 6), 17),        # 5 latent frames -> 20, 3 padding frames trimmed
    "remainder": (NARROW, (1, 4, 6, 3, 5), 20),        # 17 + a 1-latent chunk with 1 padding frame trimmed
    "three_chunks": (NARROW, (1, 4, 15, 2, 3), 51),
    "image": (NARROW, (1, 4, 1, 4, 6), 1),
    "batch2": (NARROW, (2, 4, 5, 3, 4), 17),
    "released": (RELEASED, (1, 4, 2, 4, 6), 5),
}
SAMPLES = 8000


def weights(template, name):
    """Seeded random weights for every tensor of `template` (a state dict), fp32, each seeded by the case and its key;
    ``scale`` / ``shift`` keep their released values."""
    sd = {}
    for k in sorted(template):
        if k in ("scale", "shift"):
            sd[k] = template[k].clone()
            continue
        g = torch.Generator().manual_seed(zlib.crc32(f"{name}/{k}".encode()))
        shape = template[k].shape
        if k.endswith(".bias"):
            v = 0.1 * torch.randn(shape, generator=g)
        elif len(shape) == 1:  # GroupNorm weight
            v = 1.0 + 0.2 * torch.randn(shape, generator=g)
        else:
            fan_in = int(torch.tensor(shape[1:]).prod())
            v = torch.randn(shape, generator=g) / fan_in ** 0.5
        sd[k] = v
    return sd


def latents(name, dtype=torch.float32):
    g = torch.Generator().manual_seed(4100 + list(CASES).index(name))
    return torch.randn(CASES[name][1], generator=g).to(dtype)


def sample_index(numel, name):
    g = torch.Generator().manual_seed(5100 + list(CASES).index(name))
    return torch.randperm(numel, generator=g)[:SAMPLES]


def main():
    from oracle.opensora_vae_ref import build_opensora_vae

    torch.set_grad_enabled(False)
    out = {}
    for name, (spatial, _, num_frames) in CASES.items():
        ref = build_opensora_vae(spatial)
        ref.load_state_dict(weights(ref.state_dict(), name))
        y = ref.decode(latents(name), num_frames=num_frames)
        out[f"{name}.shape"] = list(y.shape)
        flat = y.flatten()
        out[f"{name}.fp32"] = flat[sample_index(flat.numel(), name)].clone() if flat.numel() > SAMPLES else flat.clone()
        print(name, tuple(y.shape), float(y.abs().mean()))
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "opensora_vae.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
