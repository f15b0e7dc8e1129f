"""Latte VAE decode: the host logic of the SVD temporal decoder and the image VAE (layout views, zero time padding,
latent padding, the chunks of 14 frames, weight packing, the AlphaBlender weights) and of LattePipeline's decode tail on
the torch stand-ins of the kernels (tests/kernels_emul_vae_time.py), fp32, against the restated reference in
tests/golden/latte_vae.pt (oracle/gen_golden_latte_vae.py); the state-dict layout; snapshot loading; rejections; and
``generate`` around a stub denoiser."""
import json
import os

import pytest
import torch

from oracle import gen_golden_latte_vae as G
from oracle.gen_golden_opensora_vae import NARROW, weights
from tests import kernels_emul_vae_time
from videosys_b200.models.autoencoders import AutoencoderKL, AutoencoderKLTemporalDecoder


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "latte_vae.pt"))


def _vae(name):
    kind, widths, _ = G.LATTE_CASES[name]
    vae = (AutoencoderKLTemporalDecoder if kind == "temporal" else AutoencoderKL)(block_out_channels=widths).eval()
    vae.load_state_dict(weights(vae.state_dict(), "latte/" + name))
    return vae


def _pipeline(vae, dtype=torch.float32, **kw):
    """A LattePipeline built without a GPU around a stub denoiser."""
    from videosys_b200.pipelines.latte import pipeline_latte as P

    pipe = P.LattePipeline.__new__(P.LattePipeline)
    pipe._config = P.LatteConfig(vae=vae, **kw)
    pipe._device, pipe._dtype = torch.device("cpu"), dtype
    pipe.transformer = _StubTransformer()
    pipe.scheduler = P.DDIMScheduler(beta_start=0.0001, beta_end=0.02, beta_schedule="linear", variance_type="learned_range",
                                     clip_sample=False)
    pipe.vae = pipe._load_vae()
    return pipe


class _StubTransformer(torch.nn.Module):
    """Predicts 0.1 * its input (mean and learned sigma): the denoiser is not under test here."""
    config = type("C", (), dict(in_channels=4, out_channels=8, caption_channels=8))()
    parallel_manager = None

    def reset_pab_state(self):
        pass

    def forward(self, x, **kw):
        return (0.1 * torch.cat([x, x], 1),)


@pytest.mark.parametrize("name", list(G.LATTE_CASES))
def test_latte_vae_decode_vs_reference_golden(monkeypatch, gold, name):
    kernels_emul_vae_time.emulate(monkeypatch)
    pipe = _pipeline(_vae(name))
    z = G.latents("latte/" + name, G.LATTE_CASES[name][2])
    out = pipe.decode_latents_image(z) if z.shape[2] == 1 else pipe.decode_video(z)
    assert list(out.shape) == gold[f"{name}.shape"]
    flat = out.flatten()
    want = gold[f"{name}.fp32"]
    got = flat[G.sample_index(flat.numel(), name)] if flat.numel() > want.numel() else flat
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-4), (got - want).abs().max()


@pytest.mark.parametrize("name", ["temporal_16", "sd_vae"])
def test_latte_vae_state_dict_layout_matches_reference(name):
    ref = G.build_latte_vae(G.LATTE_CASES[name][0], NARROW)
    ours = _vae(name)
    assert {k: tuple(v.shape) for k, v in ref.state_dict().items()} == {k: tuple(v.shape) for k, v in ours.state_dict().items()}


def test_latte_temporal_decoder_released_keys():
    sd = AutoencoderKLTemporalDecoder().state_dict()
    for k in ("decoder.conv_in.weight", "decoder.mid_block.resnets.1.temporal_res_block.conv2.bias",
              "decoder.mid_block.attentions.0.to_out.0.weight", "decoder.mid_block.resnets.0.time_mixer.mix_factor",
              "decoder.up_blocks.2.resnets.0.spatial_res_block.conv_shortcut.weight",
              "decoder.up_blocks.0.upsamplers.0.conv.weight", "decoder.conv_out.weight", "decoder.time_conv_out.bias"):
        assert k in sd, k
    assert tuple(sd["decoder.up_blocks.3.resnets.2.temporal_res_block.conv1.weight"].shape) == (128, 128, 3, 1, 1)
    assert tuple(sd["decoder.time_conv_out.weight"].shape) == (3, 3, 3, 1, 1)
    assert not any(k.startswith(("decoder.up_blocks.3.upsamplers", "post_quant_conv")) for k in sd)


def _snapshot(tmp_path, sub, vae, cfg, drop=None):
    from safetensors.torch import save_file

    sd = {**vae.state_dict(), "encoder.conv_in.weight": torch.zeros(2), "quant_conv.weight": torch.zeros(3)}
    if drop:
        sd.pop(drop)
    d = tmp_path / sub
    d.mkdir(parents=True)
    (d / "config.json").write_text(json.dumps(cfg))
    save_file({k: v.contiguous() for k, v in sd.items()}, str(d / "diffusion_pytorch_model.safetensors"))
    return tmp_path


_TCFG = dict(_class_name="AutoencoderKLTemporalDecoder", block_out_channels=list(NARROW), layers_per_block=2,
             latent_channels=4, scaling_factor=0.18215, down_block_types=["DownEncoderBlock2D"] * 4)


def test_latte_vae_from_pretrained_local_snapshot(tmp_path):
    src = _vae("temporal_16")
    root = _snapshot(tmp_path, "vae_temporal_decoder", src, _TCFG)
    vae = AutoencoderKLTemporalDecoder.from_pretrained(str(root))
    for k, v in src.state_dict().items():
        assert torch.equal(vae.state_dict()[k], v)
    assert vae.config.block_out_channels == NARROW


def test_latte_vae_from_pretrained_missing_decoder_key_raises(tmp_path):
    root = _snapshot(tmp_path, "vae_temporal_decoder", _vae("temporal_16"), _TCFG,
                     drop="decoder.up_blocks.1.resnets.0.time_mixer.mix_factor")
    with pytest.raises(RuntimeError, match="mix_factor"):
        AutoencoderKLTemporalDecoder.from_pretrained(str(root))


def test_latte_vae_rejections():
    with pytest.raises(NotImplementedError, match="encoder"):
        AutoencoderKLTemporalDecoder(block_out_channels=NARROW).encode(torch.zeros(1, 3, 8, 8))
    with pytest.raises(ValueError, match="block_out_channels"):
        AutoencoderKLTemporalDecoder(block_out_channels=(96, 128))
    with pytest.raises(NotImplementedError, match="up_block_types"):
        AutoencoderKL(block_out_channels=NARROW, up_block_types=("UpDecoderBlock2D",) * 3 + ("AttnUpDecoderBlock2D",))
    with pytest.raises(NotImplementedError, match="mid_block_add_attention"):
        AutoencoderKL(block_out_channels=NARROW, mid_block_add_attention=False)
    with pytest.raises(NotImplementedError, match="norm_num_groups"):
        AutoencoderKL(block_out_channels=NARROW, norm_num_groups=16)
    with pytest.raises(ValueError, match="block_out_channels"):
        AutoencoderKL(block_out_channels=(128, 256, 384))


def _generate(pipe, **kw):
    return pipe.generate(prompt_embeds=torch.zeros(1, 4, 8), negative_prompt_embeds=torch.zeros(1, 4, 8), num_inference_steps=2,
                         seed=0, video_length=kw.pop("video_length", 16), height=16, width=24, verbose=False, **kw).video


def test_latte_generate_with_native_vae_instance_and_dir(monkeypatch, tmp_path):
    kernels_emul_vae_time.emulate(monkeypatch)
    vae = _vae("temporal_16")
    pipe = _pipeline(vae)
    assert pipe.vae is vae
    video = _generate(pipe)
    assert video.dtype == torch.uint8 and tuple(video.shape) == (1, 16, 16, 24, 3)
    assert int(video.max()) > int(video.min())
    # the reference's tail on the restated decoder, on the same latents
    lat = _generate(_pipeline(None))
    ref = G.build_latte_vae("temporal", NARROW)
    ref.load_state_dict(weights(ref.state_dict(), "latte/temporal_16"))
    want = G.latte_to_uint8(G.latte_decode_video(ref, lat, True))
    assert (video.int() - want.int()).abs().max() <= 1  # fp32 sums in another order may cross a uint8 step
    image = _generate(pipe, video_length=1)
    assert image.dtype == torch.float32 and tuple(image.shape) == (1, 1, 3, 16, 24)

    root = _snapshot(tmp_path / "t", "vae_temporal_decoder", vae, _TCFG)
    pipe = _pipeline(str(root))
    assert isinstance(pipe.vae, AutoencoderKLTemporalDecoder)
    sd = _vae("sd_vae")
    root = _snapshot(tmp_path / "s", "vae", sd, dict(_class_name="AutoencoderKL", block_out_channels=list(NARROW), latent_channels=4))
    pipe = _pipeline(str(root), enable_vae_temporal_decoder=False)
    assert isinstance(pipe.vae, AutoencoderKL) and pipe.vae.post_quant_conv is not None
    video = _generate(pipe, video_length=3)
    assert video.dtype == torch.uint8 and tuple(video.shape) == (1, 3, 16, 24, 3)


def test_latte_generate_vae_decode_fn_takes_precedence_and_default_returns_latents(monkeypatch):
    kernels_emul_vae_time.emulate(monkeypatch)
    calls = []
    pipe = _pipeline(_vae("temporal_16"), vae_decode_fn=lambda s: calls.append(tuple(s.shape)) or "decoded")
    assert _generate(pipe) == "decoded" and calls == [(1, 4, 16, 2, 3)]
    pipe = _pipeline(None)
    assert pipe._config.vae is None and pipe.vae is None
    lat = _generate(pipe)
    assert lat.dtype == torch.float32 and tuple(lat.shape) == (1, 4, 16, 2, 3)
