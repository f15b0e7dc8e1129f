"""CogVideoX VAE decoder: the host logic (frame batching, conv caches, context buffers, tiling and blending, weight packing)
on the torch stand-ins of the kernels (tests/kernels_emul_vae.py), fp32, against the outputs of the UNMODIFIED reference
decoder in tests/golden/cogvideox_vae.pt (oracle/gen_golden_cogvideox_vae.py); the state-dict layout against the
reference; the rejections; and the pipeline's decode stage."""
import json
import os

import pytest
import torch

from oracle import ref_loader
from oracle.gen_golden_cogvideox_vae import CASES, latents, sample_index, weights
from tests import kernels_emul_vae
from videosys_b200.models.autoencoders import AutoencoderKLCogVideoX


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "cogvideox_vae.pt"))


def _vae(name):
    cfg, _, tiling = CASES[name]
    vae = AutoencoderKLCogVideoX(**cfg).eval()
    vae.load_state_dict(weights(vae.state_dict(), name))
    if tiling is not None:
        vae.enable_tiling(**tiling)
    return vae


@pytest.mark.parametrize("name", list(CASES))
def test_cogvideox_vae_decode_vs_reference_golden(monkeypatch, gold, name):
    kernels_emul_vae.emulate(monkeypatch)
    out = _vae(name).decode(latents(name)).sample
    assert list(out.shape) == gold[f"{name}.shape"]
    flat = out.flatten()
    want = gold[f"{name}.fp32"]
    got = flat[sample_index(flat.numel(), name)] if flat.numel() > want.numel() else flat
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-4), (got - want).abs().max()


def test_cogvideox_vae_slicing_and_cache_reset(monkeypatch):
    """enable_slicing decodes sample by sample to the same values; a second decode starts from cleared conv caches."""
    kernels_emul_vae.emulate(monkeypatch)
    vae = _vae("small_f4_b2")
    z = latents("small_f4_b2")
    a = vae.decode(z).sample
    vae.enable_slicing()
    b = vae.decode(z).sample
    vae.disable_slicing()
    assert torch.allclose(a, b, rtol=1e-4, atol=1e-4)  # fp32 CPU convolutions sum in a batch-size dependent order
    assert all(m.conv_cache is None for m in vae.modules() if hasattr(m, "conv_cache"))


def test_cogvideox_vae_state_dict_round_trip_with_reference():
    if not ref_loader.available():
        pytest.skip("reference checkout not present")
    from oracle.cogvideox_vae_ref import build_cogvideox_vae

    for name in ("small_f3", "released_f3"):
        cfg = CASES[name][0]
        ref = build_cogvideox_vae(**cfg)
        ours = AutoencoderKLCogVideoX(**cfg)
        rs = ref.state_dict()
        dec = {k: tuple(v.shape) for k, v in rs.items() if k.startswith("decoder.")}
        assert dec == {k: tuple(v.shape) for k, v in ours.state_dict().items()}
        assert all(k.startswith(("decoder.", "encoder.", "quant_conv.")) for k in rs)
        ours.load_state_dict(weights(rs, name), strict=True)  # the full reference dict: encoder.* dropped
        ref.load_state_dict({**rs, **ours.state_dict()}, strict=True)
        for k, v in ours.state_dict().items():
            assert torch.equal(ref.state_dict()[k], v)


def test_cogvideox_vae_load_state_dict_is_strict_about_the_decoder():
    vae = AutoencoderKLCogVideoX(**CASES["small_f3"][0])
    sd = vae.state_dict()
    sd["encoder.conv_in.conv.weight"] = torch.zeros(1)  # dropped by rule
    vae.load_state_dict(sd)
    bad = dict(sd)
    bad.pop("decoder.conv_out.conv.bias")
    with pytest.raises(RuntimeError, match="conv_out"):
        vae.load_state_dict(bad)
    with pytest.raises(RuntimeError, match="Unexpected"):
        vae.load_state_dict({**sd, "decoder.extra.weight": torch.zeros(1)})


def test_cogvideox_vae_from_pretrained_local_snapshot(tmp_path):
    cfg = dict(CASES["small_f3"][0], _class_name="AutoencoderKLCogVideoX")
    (tmp_path / "vae").mkdir()
    (tmp_path / "vae" / "config.json").write_text(json.dumps(cfg))
    src = AutoencoderKLCogVideoX(**CASES["small_f3"][0])
    sd = weights(src.state_dict(), "small_f3")
    torch.save({**sd, "encoder.conv_in.conv.weight": torch.zeros(2)}, tmp_path / "vae" / "diffusion_pytorch_model.bin")
    vae = AutoencoderKLCogVideoX.from_pretrained(str(tmp_path), subfolder="vae")
    assert vae.config.block_out_channels == (64, 64, 128, 128)
    assert torch.equal(vae.state_dict()["decoder.conv_out.conv.weight"], sd["decoder.conv_out.conv.weight"])


def test_cogvideox_vae_rejections():
    with pytest.raises(NotImplementedError):
        AutoencoderKLCogVideoX(use_post_quant_conv=True)
    with pytest.raises(NotImplementedError, match="encoder"):
        AutoencoderKLCogVideoX(**CASES["small_f3"][0]).encode(torch.zeros(1, 3, 1, 8, 8))
    with pytest.raises(ValueError, match="block_out_channels"):
        AutoencoderKLCogVideoX(block_out_channels=(96, 96, 128, 128))
    with pytest.raises(ValueError, match="norm_num_groups"):
        AutoencoderKLCogVideoX(block_out_channels=(64, 64, 128, 128), norm_num_groups=48)
    with pytest.raises(ValueError, match="latent_channels"):
        AutoencoderKLCogVideoX(block_out_channels=(64, 64, 128, 128), latent_channels=8)
    with pytest.raises(ValueError, match="out_channels"):
        AutoencoderKLCogVideoX(block_out_channels=(64, 64, 128, 128), out_channels=4)
    with pytest.raises(ValueError, match="up_block_type"):
        AutoencoderKLCogVideoX(up_block_types=("UpDecoderBlock2D",) * 4)


def _pipeline(monkeypatch, vae, vae_tiling=False):
    """A CogVideoXPipeline with a tiny transformer whose noise prediction is zero, built without a GPU."""
    from videosys_b200.pipelines.cogvideox import pipeline_cogvideox as P

    class _ZeroDiT(torch.nn.Module):
        config = type("C", (), dict(in_channels=16, text_embed_dim=8, use_rotary_positional_embeddings=False, patch_size=2))()

        def reset_pab_state(self):
            pass

        def forward(self, hidden_states, **kw):
            return (torch.zeros_like(hidden_states),)

    pipe = P.CogVideoXPipeline.__new__(P.CogVideoXPipeline)
    pipe._config = P.CogVideoXConfig(vae=vae, vae_tiling=vae_tiling)
    pipe._device, pipe._dtype = torch.device("cpu"), torch.float32
    pipe.transformer = _ZeroDiT()
    pipe.scheduler = P.CogVideoXDDIMScheduler()
    pipe.vae = pipe._load_vae()
    monkeypatch.setattr(pipe, "_maybe_seed", lambda seed: None, raising=False)
    return pipe


@pytest.mark.parametrize("output_type", ["pt", "np", "pil", "latent"])
def test_cogvideox_generate_with_native_vae_returns_reference_shapes(monkeypatch, output_type):
    kernels_emul_vae.emulate(monkeypatch)
    vae = _vae("small_f3")
    pipe = _pipeline(monkeypatch, vae)
    pe = torch.randn(1, 4, 8)
    out = pipe.generate(height=48, width=80, num_frames=9, num_inference_steps=2, guidance_scale=1.0, prompt_embeds=pe,
                        output_type=output_type).video
    if output_type == "pt":
        assert tuple(out.shape) == (1, 9, 3, 48, 80)  # 4 (3 - 1) + 1 frames
        assert float(out.min()) >= 0 and float(out.max()) <= 1
    elif output_type == "np":
        assert out.shape == (1, 9, 48, 80, 3)
    elif output_type == "pil":
        assert len(out) == 1 and len(out[0]) == 9 and out[0][0].size == (80, 48)
    else:
        assert tuple(out.shape) == (1, 3, 16, 6, 10)


def test_cogvideox_generate_without_vae_returns_latents(monkeypatch):
    kernels_emul_vae.emulate(monkeypatch)
    pipe = _pipeline(monkeypatch, None)
    assert pipe.vae is None
    out = pipe.generate(height=48, width=80, num_frames=9, num_inference_steps=2, guidance_scale=1.0,
                        prompt_embeds=torch.randn(1, 4, 8), output_type="pt").video
    assert tuple(out.shape) == (1, 3, 16, 6, 10)


def test_cogvideox_generate_vae_matches_reference_tail(monkeypatch):
    """The decode stage equals the reference tail: permute, / scaling_factor, decode, (x / 2 + 0.5).clamp(0, 1)."""
    kernels_emul_vae.emulate(monkeypatch)
    vae = _vae("small_f3")
    pipe = _pipeline(monkeypatch, vae, vae_tiling=True)
    assert vae.use_tiling
    lat = torch.randn(1, 3, 16, 6, 10)
    got = pipe.decode_latents_to_video(lat, "pt")
    want = (vae.decode(1 / vae.config.scaling_factor * lat.permute(0, 2, 1, 3, 4)).sample / 2 + 0.5).clamp(0, 1).permute(0, 2, 1, 3, 4)
    assert torch.allclose(got, want, atol=1e-6)
