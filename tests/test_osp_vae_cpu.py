"""Open-Sora-Plan causal-VAE decoder (v1.1.0 and v1.2.0): the host logic (context buffers, latent padding, attention
layouts, up-samplers, tiling and blending, weight packing) on the torch stand-ins of the kernels
(tests/kernels_emul_vae.py), fp32, against the outputs of the UNMODIFIED reference decoders in tests/golden/osp_vae.pt
(oracle/gen_golden_osp_vae.py); the state-dict layout against the reference; checkpoint loading; the rejections; and the
pipeline's decode stage."""
import json
import os

import pytest
import torch

from oracle import ref_loader
from oracle.gen_golden_osp_vae import CASES, V110_RES, V120, apply_tiling, latents, sample_index, weights
from tests import kernels_emul_vae
from videosys_b200.models.autoencoders import CausalVAEModelV110, CausalVAEModelV120
from videosys_b200.models.autoencoders.autoencoder_kl_open_sora_plan import decoder_class


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "osp_vae.pt"))


def _vae(name):
    version, cfg, _, tiling = CASES[name]
    vae = decoder_class(version)(**cfg).eval()
    vae.load_state_dict(weights(vae.state_dict(), name))
    if tiling is not None:
        apply_tiling(vae, tiling)
    return vae


def _check(out, gold, name):
    assert list(out.shape) == gold[f"{name}.shape"]
    flat = out.flatten()
    want = gold[f"{name}.fp32"]
    got = flat[sample_index(flat.numel(), name)] if flat.numel() > want.numel() else flat
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-4), (got - want).abs().max()


@pytest.mark.parametrize("name", list(CASES))
def test_osp_vae_decode_vs_reference_golden(monkeypatch, gold, name):
    kernels_emul_vae.emulate(monkeypatch)
    _check(_vae(name).decode(latents(name)), gold, name)


def test_osp_vae_tiled_case_really_tiles(monkeypatch):
    """The tiled golden case runs several time chunks and overlapping tiles; untiled it decodes to the same shape."""
    kernels_emul_vae.emulate(monkeypatch)
    vae = _vae("v110_tiled")
    calls = []
    orig = vae._decode_tile
    monkeypatch.setattr(vae, "_decode_tile", lambda z: calls.append(tuple(z.shape)) or orig(z))
    tiled = vae.decode(latents("v110_tiled"))
    assert len(calls) == 2 * 2 * 3 and {c[2] for c in calls} == {3}
    vae.disable_tiling()
    assert vae.decode(latents("v110_tiled")).shape == tiled.shape


@pytest.mark.parametrize("version,cfg", [("v120", V120), ("v110", V110_RES), ("v110", CASES["v110_default_f3"][1])])
def test_osp_vae_state_dict_round_trip_with_reference(version, cfg):
    if not ref_loader.available():
        pytest.skip("reference checkout not present")
    from oracle.osp_vae_ref import build_osp_vae

    ref = build_osp_vae(version, **cfg)
    ours = decoder_class(version)(**cfg)
    rs = ref.state_dict()
    kept = {k: tuple(v.shape) for k, v in rs.items() if k.startswith(("decoder.", "post_quant_conv."))}
    assert kept == {k: tuple(v.shape) for k, v in ours.state_dict().items()}
    assert all(k.startswith(("decoder.", "post_quant_conv.", "encoder.", "quant_conv.")) for k in rs)
    ours.load_state_dict(weights(rs, "v120_f3"), strict=True)  # the full reference dict: encoder.* / quant_conv.* dropped
    ref.load_state_dict({**rs, **ours.state_dict()}, strict=True)
    for k, v in ours.state_dict().items():
        assert torch.equal(ref.state_dict()[k], v)


def test_osp_vae_load_state_dict_is_strict_about_the_decoder():
    vae = CausalVAEModelV120(**V120)
    sd = vae.state_dict()
    vae.load_state_dict({**sd, "encoder.conv_in.conv.weight": torch.zeros(1), "quant_conv.conv.bias": torch.zeros(1),
                         "loss.logvar": torch.zeros(1)})
    bad = dict(sd)
    bad.pop("post_quant_conv.conv.bias")
    with pytest.raises(RuntimeError, match="post_quant_conv"):
        vae.load_state_dict(bad)
    with pytest.raises(RuntimeError, match="Unexpected"):
        vae.load_state_dict({**sd, "decoder.extra.weight": torch.zeros(1)})


def _snapshot(tmp_path, cls, cfg, name):
    src = cls(**cfg)
    sd = weights(src.state_dict(), name)
    d = tmp_path / "vae"
    d.mkdir()
    (d / "config.json").write_text(json.dumps(dict(cfg, _class_name="CausalVAEModel")))
    return d, sd


@pytest.mark.parametrize("nesting", ["flat", "state_dict", "gen_model", "ema"])
def test_osp_vae_v120_from_pretrained_ckpt(tmp_path, monkeypatch, nesting):
    monkeypatch.delenv("NOT_USE_EMA_MODEL", raising=False)
    d, sd = _snapshot(tmp_path, CausalVAEModelV120, V120, "v120_f3")
    full = {**sd, "encoder.conv_in.conv.weight": torch.zeros(2), "loss.discriminator.w": torch.zeros(2)}
    blob = {"flat": full, "state_dict": {"state_dict": full}, "gen_model": {"state_dict": {"gen_model": full}},
            "ema": {"ema_state_dict": {"module." + k: v for k, v in full.items()},
                    "state_dict": {k: torch.zeros_like(v) for k, v in full.items()}}}[nesting]
    torch.save(blob, d / "checkpoint.ckpt")
    vae = CausalVAEModelV120.from_pretrained(str(tmp_path), subfolder="vae")
    assert vae.config.hidden_size == 64
    for k in ("decoder.conv_out.conv.weight", "post_quant_conv.conv.bias", "decoder.mid.attn_1.q.conv.weight"):
        assert torch.equal(vae.state_dict()[k], sd[k])


def test_osp_vae_v110_from_pretrained_ckpt_and_diffusers_weights(tmp_path):
    d, sd = _snapshot(tmp_path, CausalVAEModelV110, V110_RES, "v110_res_attn3d_b2")
    torch.save({**sd, "encoder.conv_in.conv.weight": torch.zeros(2)}, d / "diffusion_pytorch_model.bin")
    vae = CausalVAEModelV110.from_pretrained(str(tmp_path), subfolder="vae")  # no *.ckpt: the diffusers-style weights
    assert torch.equal(vae.state_dict()["decoder.up.2.time_upsample.mix_factor"], sd["decoder.up.2.time_upsample.mix_factor"])
    sd2 = {k: v + 1 for k, v in sd.items()}
    torch.save({"state_dict": sd2}, d / "last.ckpt")  # a *.ckpt takes precedence
    vae = CausalVAEModelV110.from_pretrained(str(d))
    assert torch.equal(vae.state_dict()["decoder.conv_in.conv.weight"], sd2["decoder.conv_in.conv.weight"])
    with pytest.raises(FileNotFoundError):
        CausalVAEModelV120.from_pretrained(str(tmp_path / "missing"))


@pytest.mark.parametrize("version,kw,exc,match", [
    ("v110", dict(decoder_attention="AttnBlock"), NotImplementedError, "AttnBlock"),
    ("v110", dict(decoder_attention="LinAttnBlock"), NotImplementedError, "LinAttnBlock"),
    ("v110", dict(decoder_attention="TemporalAttnBlock"), NotImplementedError, "TemporalAttnBlock"),
    ("v110", dict(decoder_temporal_upsample=("", "", "", "TimeUpsampleResAdv2x")), NotImplementedError, "TimeUpsampleResAdv2x"),
    ("v110", dict(decoder_spatial_upsample=("", "Upsample", "Upsample", "Upsample")), NotImplementedError, "Upsample"),
    ("v110", dict(decoder_resnet_blocks=("ResnetBlock2D",) * 4), NotImplementedError, "ResnetBlock2D"),
    ("v110", dict(attn_resolutions=(16,)), NotImplementedError, "attn_resolutions"),
    ("v120", {}, NotImplementedError, "AttnBlock3D"),  # the v1.2.0 defaults name modules its file does not define
    ("v120", dict(V120, decoder_temporal_upsample=("", "", "", "TimeUpsampleRes2x")), NotImplementedError, "TimeUpsampleRes2x"),
    ("v110", dict(hidden_size=96), ValueError, "hidden_size"),
    ("v110", dict(hidden_size=64, hidden_size_mult=(1, 2, 4, 16)), ValueError, "hidden_size"),
    ("v110", dict(z_channels=32), ValueError, "z_channels"),
])
def test_osp_vae_rejections(version, kw, exc, match):
    with pytest.raises(exc, match=match):
        decoder_class(version)(**kw)


def test_osp_vae_encode_is_out_of_scope():
    with pytest.raises(NotImplementedError, match="encoder"):
        CausalVAEModelV110(hidden_size=64, num_res_blocks=1).encode(torch.zeros(1, 3, 1, 8, 8))


def _pipeline(monkeypatch, vae, enable_tiling=False):
    """A v1.1.0 OpenSoraPlanPipeline with a tiny transformer whose noise prediction is zero, built without a GPU."""
    from videosys_b200.pipelines.open_sora_plan import pipeline_open_sora_plan as P

    class _ZeroDiT(torch.nn.Module):
        config = type("C", (), dict(in_channels=4, out_channels=4, caption_channels=8))()
        video_length = 3

        def reset_pab_state(self):
            pass

        def forward(self, hidden_states, **kw):
            return (torch.zeros_like(hidden_states),)

    pipe = P.OpenSoraPlanPipeline.__new__(P.OpenSoraPlanPipeline)
    pipe._config = P.OpenSoraPlanConfig(version="v110", transformer_type="65x512x512", vae=vae, enable_tiling=enable_tiling,
                                        transformer_config={})
    pipe._config.num_frames = 7
    pipe._device, pipe._dtype = torch.device("cpu"), torch.float32
    pipe.transformer = _ZeroDiT()
    pipe.scheduler = P.PNDMScheduler()
    pipe.vae = pipe._load_vae()
    monkeypatch.setattr(pipe, "_maybe_seed", lambda seed: None, raising=False)
    return pipe


def _generate(pipe, output_type="pil"):
    """Latents and caption from a local generator: the global RNG state of the test process is left alone."""
    g = torch.Generator().manual_seed(0)
    return pipe.generate(height=24, width=40, num_inference_steps=4, guidance_scale=1.0, latents=torch.randn(1, 4, 3, 3, 5, generator=g),
                         prompt_embeds=torch.randn(1, 4, 8, generator=g), output_type=output_type).video


def test_osp_generate_with_native_vae_matches_reference_tail(monkeypatch):
    kernels_emul_vae.emulate(monkeypatch)
    vae = _vae("v110_default_f3")
    pipe = _pipeline(monkeypatch, vae)
    video = _generate(pipe)
    lat = _generate(pipe, "latents")
    assert video.dtype == torch.uint8 and tuple(video.shape) == (1, 7, 24, 40, 3)  # 9 decoded frames cut to num_frames
    dec = vae.decode(lat / 0.18215).permute(0, 2, 1, 3, 4)
    want = ((dec / 2.0 + 0.5).clamp(0, 1) * 255).to(torch.uint8).permute(0, 1, 3, 4, 2)[:, :7, :24, :40]
    assert torch.equal(video, want)


def test_osp_generate_without_vae_returns_the_same_latents(monkeypatch):
    kernels_emul_vae.emulate(monkeypatch)
    with_vae = _generate(_pipeline(monkeypatch, _vae("v110_default_f3")), "latents")
    pipe = _pipeline(monkeypatch, None)
    assert pipe.vae is None
    lat = _generate(pipe, "pil")
    assert tuple(lat.shape) == (1, 4, 3, 3, 5) and lat.dtype == torch.float32
    assert torch.equal(lat, with_vae)


def test_osp_pipeline_applies_the_reference_tiling(monkeypatch, tmp_path):
    kernels_emul_vae.emulate(monkeypatch)
    pipe = _pipeline(monkeypatch, _vae("v110_default_f3"), enable_tiling=True)
    v = pipe.vae
    assert v.use_tiling and (v.tile_sample_min_size, v.tile_latent_min_size, v.tile_sample_min_size_t, v.tile_latent_min_size_t) == \
        (512, 64, 29, 8) and v.tile_overlap_factor == 0.25
    d, sd = _snapshot(tmp_path, CausalVAEModelV110, CASES["v110_default_f3"][1], "v110_default_f3")
    torch.save({"state_dict": sd}, d / "checkpoint.ckpt")
    pipe = _pipeline(monkeypatch, str(tmp_path))  # a snapshot root with a vae/ folder
    assert isinstance(pipe.vae, CausalVAEModelV110) and not pipe.vae.use_tiling
