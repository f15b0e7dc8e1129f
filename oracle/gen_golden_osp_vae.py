"""Writes tests/golden/osp_vae.pt: outputs of the UNMODIFIED reference Open-Sora-Plan causal-VAE decoders
(oracle/osp_vae_ref.py, v1.1.0 and v1.2.0) in fp32 on the CPU.

    python -m oracle.gen_golden_osp_vae

Only outputs are stored.  Weights and latents are regenerated from seeds by a CPU generator (``weights`` / ``latents``
below).  Outputs are stored at a seeded random subset of ``SAMPLES`` elements (``sample_index``), plus their shape.  The
weights are random rather than the reference's init (which zeroes every convolution bias and leaves the GroupNorm affine
parameters at 1 / 0, hiding bias and channel-order bugs); each tensor is seeded by its name, so the reference's full state
dict and the decoder-only one get the same values.
"""
import os
import zlib

import torch

_V120_ENCODER = dict(encoder_attention="AttnBlock3DFix", encoder_spatial_downsample=("Downsample", "Downsample", "Downsample", ""),
                     encoder_temporal_downsample=("", "", "", ""))
V120 = dict(_V120_ENCODER, hidden_size=64, hidden_size_mult=(1, 2, 4, 4), num_res_blocks=1, decoder_attention="AttnBlock3DFix",
            decoder_resnet_blocks=("ResnetBlock3D", "ResnetBlock3D_GC", "ResnetBlock3D", "ResnetBlock3D"),
            decoder_spatial_upsample=("", "SpatialUpsample2x", "Spatial2xTime2x3DUpsample", "Spatial2xTime2x3DUpsample"),
            decoder_temporal_upsample=("", "", "", ""), use_quant_layer=True)
V120_CONV2D = dict(V120, decoder_conv_in="Conv2d", decoder_conv_out="Conv2d", use_quant_layer=False)
V110_RES = dict(hidden_size=64, hidden_size_mult=(1, 2, 4, 4), num_res_blocks=1, decoder_attention="AttnBlock3D",
                decoder_temporal_upsample=("", "", "TimeUpsampleRes2x", "TimeUpsampleRes2x"))
V110_DEFAULT = dict(hidden_size=64, num_res_blocks=1)
V110_FIX = dict(V110_RES, decoder_attention="AttnBlock3DFix")
V120_RELEASED = dict(_V120_ENCODER, decoder_attention="AttnBlock3DFix",
                     decoder_spatial_upsample=("", "SpatialUpsample2x", "Spatial2xTime2x3DUpsample", "Spatial2xTime2x3DUpsample"),
                     decoder_temporal_upsample=("", "", "", ""))

# name -> (version, constructor keywords, latent shape [B, C, T, h, w], tiling attributes or None)
CASES = {
    "v120_f3": ("v120", V120, (1, 4, 3, 4, 6), None),                 # Spatial2xTime2x3DUpsample over 3 latent frames
    "v120_f1": ("v120", V120, (1, 4, 1, 4, 6), None),                 # its T = 1 branch
    "v120_conv2d_f2": ("v120", V120_CONV2D, (1, 4, 2, 3, 5), None),   # Conv2d conv_in / conv_out, no post_quant_conv, P = 15
    "v110_res_attn3d_b2": ("v110", V110_RES, (2, 4, 3, 4, 6), None),  # AttnBlock3D's frame / channel mixing, two samples
    "v110_default_f3": ("v110", V110_DEFAULT, (1, 4, 3, 4, 6), None),  # constructor defaults: TimeUpsample2x
    "v110_tiled": ("v110", V110_FIX, (1, 4, 5, 6, 7),                  # 2 time chunks, 2 x 3 blended tiles
                   dict(tile_latent_min_size=4, tile_sample_min_size=32, tile_latent_min_size_t=3, tile_sample_min_size_t=9,
                        tile_overlap_factor=0.25)),
    "v120_released": ("v120", V120_RELEASED, (1, 4, 2, 4, 4), None),  # hidden 128, C = 512 attention
}
SAMPLES = 8000


def weights(template, name):
    """Seeded random weights for every tensor of `template` (a state dict), fp32, each seeded by the case and its key."""
    sd = {}
    for k in sorted(template):
        g = torch.Generator().manual_seed(zlib.crc32(f"{name}/{k}".encode()))
        shape = template[k].shape
        leaf = k.rsplit(".", 2)
        if leaf[-1] == "mix_factor":
            v = torch.randn(shape, generator=g)
        elif leaf[-2].startswith("norm") and leaf[-1] == "weight":
            v = 1.0 + 0.2 * torch.randn(shape, generator=g)
        elif leaf[-1] == "bias":
            v = 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = int(torch.tensor(shape[1:]).prod())
            v = torch.randn(shape, generator=g) / fan_in ** 0.5
        sd[k] = v
    return sd


def latents(name, dtype=torch.float32):
    g = torch.Generator().manual_seed(2100 + list(CASES).index(name))
    return torch.randn(CASES[name][2], generator=g).to(dtype)


def sample_index(numel, name):
    g = torch.Generator().manual_seed(3100 + list(CASES).index(name))
    return torch.randperm(numel, generator=g)[:SAMPLES]


def apply_tiling(vae, tiling):
    vae.enable_tiling()
    for k, v in tiling.items():
        setattr(vae, k, v)


def main():
    from oracle.osp_vae_ref import build_osp_vae

    torch.set_grad_enabled(False)
    out = {}
    for name, (version, cfg, _, tiling) in CASES.items():
        ref = build_osp_vae(version, **cfg)
        ref.load_state_dict(weights(ref.state_dict(), name))
        if tiling is not None:
            apply_tiling(ref, tiling)
        y = ref.decode(latents(name))
        out[f"{name}.shape"] = list(y.shape)
        flat = y.flatten()
        out[f"{name}.fp32"] = flat[sample_index(flat.numel(), name)].clone() if flat.numel() > SAMPLES else flat.clone()
        print(name, tuple(y.shape), float(y.abs().mean()))
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "osp_vae.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
