"""Writes tests/golden/cogvideox_vae.pt: outputs of the UNMODIFIED reference CogVideoX VAE decoder
(oracle/cogvideox_vae_ref.py) in fp32 on the CPU.

    python -m oracle.gen_golden_cogvideox_vae

Only outputs are stored.  Weights and latents are regenerated from seeds by a CPU generator (``weights`` / ``latents``
below).  Large outputs are stored at a seeded random subset of ``SAMPLES`` elements (``sample_index``), plus their shape.
The weights are random rather than the reference's init, scaled by 1 / sqrt(fan-in) so that the activations stay O(1):
the init would leave the GroupNorm affine parameters at 1 / 0, which hides channel-order bugs.
"""
import os

import torch

# name -> (constructor keywords, latent shape [B, C, T, h, w], enable_tiling keywords or None)
SMALL = dict(block_out_channels=(64, 64, 128, 128), layers_per_block=1, norm_num_groups=32, sample_height=48, sample_width=80)
CASES = {
    "small_f3": (SMALL, (1, 16, 3, 6, 10), None),     # one frame batch of 3
    "small_f4_b2": (SMALL, (2, 16, 4, 6, 10), None),  # 2 + 2 frames, conv caches carried; two samples
    "small_f5": (SMALL, (1, 16, 5, 6, 10), None),     # 3 + 2 frames
    "small_tiled": (SMALL, (1, 16, 3, 8, 12), dict(tile_sample_min_height=48, tile_sample_min_width=64)),
    "released_f3": (dict(block_out_channels=(128, 256, 256, 512), layers_per_block=3), (1, 16, 3, 4, 6), None),
}
SAMPLES = 20000


def weights(template, name):
    """Seeded random weights for every tensor of `template` (a state dict), fp32."""
    g = torch.Generator().manual_seed(1000 + list(CASES).index(name))
    sd = {}
    for k in sorted(template):
        shape = template[k].shape
        if k.endswith("norm_layer.weight"):
            v = 1.0 + 0.2 * torch.randn(shape, generator=g)
        elif k.endswith("bias"):
            v = 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = int(torch.tensor(shape[1:]).prod())
            v = torch.randn(shape, generator=g) / fan_in ** 0.5
        sd[k] = v
    return sd


def latents(name, dtype=torch.float32):
    g = torch.Generator().manual_seed(2000 + list(CASES).index(name))
    return torch.randn(CASES[name][1], generator=g).to(dtype)


def sample_index(numel, name):
    g = torch.Generator().manual_seed(3000 + list(CASES).index(name))
    return torch.randperm(numel, generator=g)[:SAMPLES]


def main():
    from oracle.cogvideox_vae_ref import build_cogvideox_vae

    torch.set_grad_enabled(False)
    out = {}
    for name, (cfg, _, tiling) in CASES.items():
        ref = build_cogvideox_vae(**cfg)
        ref.load_state_dict(weights(ref.state_dict(), name))
        if tiling is not None:
            ref.enable_tiling(**tiling)
        y = ref.decode(latents(name)).sample
        out[f"{name}.shape"] = list(y.shape)
        flat = y.flatten()
        out[f"{name}.fp32"] = flat[sample_index(flat.numel(), name)].clone() if flat.numel() > SAMPLES else flat.clone()
        print(name, tuple(y.shape), float(y.abs().mean()))
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "cogvideox_vae.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
