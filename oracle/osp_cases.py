"""TEST INFRASTRUCTURE ONLY -- Open-Sora-Plan v1.1.0 parity cases shared by oracle/gen_golden_osp.py (which runs the
UNMODIFIED reference model on them, authoring container) and tests/test_osp_gpu.py (which runs the native product on the same
seeded inputs and weights and compares with the stored reference outputs)."""
import torch

from . import synth

BASE = dict(in_channels=4, out_channels=8, attention_bias=True, patch_size=2, activation_fn="gelu-approximate",
            norm_type="ada_norm_single", norm_elementwise_affine=False, norm_eps=1e-6, attention_mode="math")
CASES = {
    # name: (model config, latent [B, C, F, H, W], text tokens, timestep)
    "small_rope": (dict(BASE, num_attention_heads=2, attention_head_dim=72, num_layers=2, cross_attention_dim=144,
                        sample_size=(8, 8), caption_channels=32, video_length=5, use_rope=True), (2, 4, 5, 8, 8), 7, 500),
    "small_norope": (dict(BASE, num_attention_heads=2, attention_head_dim=72, num_layers=2, cross_attention_dim=144,
                          sample_size=(8, 8), caption_channels=32, video_length=5, use_rope=False), (2, 4, 5, 8, 8), 7, 500),
    # the released model's width (16 heads x 72 = 1152, 4096-wide captions, 17 latent frames = 65 video frames), 2 of its 28
    # layers, a 24 x 24 latent (144 patches per frame; 512 x 512 video would be 64 x 64)
    "wide_rope": (dict(BASE, num_attention_heads=16, attention_head_dim=72, num_layers=2, cross_attention_dim=1152,
                       sample_size=(24, 24), caption_channels=4096, video_length=17, use_rope=True), (2, 4, 17, 24, 24), 40, 300),
}
PAB_TIMESTEPS = [900, 700, 650, 600, 550, 500, 450, 50]
PAB_KW = dict(spatial_broadcast=True, spatial_threshold=[100, 850], spatial_range=2, temporal_broadcast=True,
              temporal_threshold=[100, 850], temporal_range=3, cross_broadcast=True, cross_threshold=[100, 850], cross_range=4,
              mlp_broadcast=True, mlp_spatial_broadcast_config={700: {"block": [0, 1], "skip_count": 2}, 550: {"block": [1], "skip_count": 1}},
              mlp_temporal_broadcast_config={700: {"block": [0, 1], "skip_count": 2}, 550: {"block": [1], "skip_count": 1}})


def weights(state_dict, name, dtype):
    sd = synth.fill_state_dict({k: v.float() for k, v in state_dict.items()}, f"ospg.{name}.")
    return {k: v.to(dtype) if v.is_floating_point() else v for k, v in sd.items()}


def inputs(name, dtype, step=None):
    cfg, shape, L, t = CASES[name]
    tag = f"ospg.{name}." + ("" if step is None else f"s{step}.")
    x = synth.normalish(tag + "x", shape).to(dtype)
    enc = synth.normalish(tag + "enc", (shape[0], 1, L, cfg["caption_channels"])).to(dtype)
    m = torch.ones(shape[0], 1, L)
    m[shape[0] - 1, 0, L - max(2, L // 4):] = 0  # tokenizer padding on the last sample
    return x, enc, m, torch.tensor([t] * shape[0])


# ---- Open-Sora-Plan v1.2.0 (OpenSoraT2V) ------------------------------------------------------------------------------------------
BASE12 = dict(in_channels=4, out_channels=8, attention_bias=True, patch_size=2, patch_size_t=1, activation_fn="gelu-approximate",
              norm_type="ada_norm_single", norm_elementwise_affine=False, norm_eps=1e-6, attention_mode="math", downsampler=None)
CASES12 = {
    "small_rope": (dict(BASE12, num_attention_heads=2, attention_head_dim=96, num_layers=2, cross_attention_dim=192, sample_size=(8, 8),
                        sample_size_t=5, caption_channels=32, interpolation_scale_h=1.0, interpolation_scale_w=2.0,
                        interpolation_scale_t=1.5, use_rope=True), (2, 4, 5, 8, 8), 7, 500),
    "small_abspos": (dict(BASE12, num_attention_heads=2, attention_head_dim=96, num_layers=2, cross_attention_dim=192,
                          sample_size=(8, 8), sample_size_t=5, caption_channels=32, use_rope=False), (2, 4, 5, 8, 8), 7, 500),
    # the released model's width (24 heads x 96 = 2304, 4096-wide captions), 2 of its 32 layers, 4 latent frames of 12 x 16
    # latent pixels (48 patches per frame: 192 tokens; 29x480p would be 8 x 30 x 40 = 9600)
    "wide_rope": (dict(BASE12, num_attention_heads=24, attention_head_dim=96, num_layers=2, cross_attention_dim=2304,
                       sample_size=(12, 16), sample_size_t=4, caption_channels=4096, interpolation_scale_h=1.0,
                       interpolation_scale_w=1.0, interpolation_scale_t=1.0, use_rope=True), (2, 4, 4, 12, 16), 40, 300),
}
PAB12_KW = dict(spatial_broadcast=True, spatial_threshold=[100, 850], spatial_range=2, cross_broadcast=True,
                cross_threshold=[100, 850], cross_range=3)


def inputs12(name, dtype, step=None):
    cfg, shape, L, t = CASES12[name]
    tag = f"ospg12.{name}." + ("" if step is None else f"s{step}.")
    x = synth.normalish(tag + "x", shape).to(dtype)
    enc = synth.normalish(tag + "enc", (shape[0], 1, L, cfg["caption_channels"])).to(dtype)
    m = torch.ones(shape[0], 1, L)
    m[shape[0] - 1, 0, L - max(2, L // 4):] = 0
    return x, enc, m, torch.tensor([t] * shape[0])
