"""OpenSora v1.2 VAE decoder: the host logic (micro-frame chunks, time padding and trim, zero causal context, the
depth-to-time shuffle, latent padding, image micro-batches, weight packing) on the torch stand-ins of the kernels
(tests/kernels_emul_vae.py), fp32, against the outputs of the UNMODIFIED reference decode in
tests/golden/opensora_vae.pt (oracle/gen_golden_opensora_vae.py); the state-dict layout against the reference and the
restated SDXL decoder; snapshot loading; and the pipeline's decode stage."""
import os

import pytest
import torch

from oracle import ref_loader
from oracle.gen_golden_opensora_vae import CASES, NARROW, latents, sample_index, weights
from tests import kernels_emul_vae
from videosys_b200.models.autoencoders import VideoAutoencoderPipeline


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "opensora_vae.pt"))


def _vae(name, **kw):
    vae = VideoAutoencoderPipeline(spatial_block_out_channels=CASES[name][0], **kw).eval()
    vae.load_state_dict(weights(vae.state_dict(), name))
    return vae


@pytest.mark.parametrize("name", list(CASES))
def test_opensora_vae_decode_vs_reference_golden(monkeypatch, gold, name):
    kernels_emul_vae.emulate(monkeypatch)
    out = _vae(name).decode(latents(name), num_frames=CASES[name][2])
    assert list(out.shape) == gold[f"{name}.shape"]
    flat = out.flatten()
    want = gold[f"{name}.fp32"]
    got = flat[sample_index(flat.numel(), name)] if flat.numel() > want.numel() else flat
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-4), (got - want).abs().max()


def test_opensora_vae_micro_batches_do_not_change_the_result(monkeypatch):
    """Each image is its own GroupNorm sample: one spatial pass per frame or all frames at once decode alike."""
    kernels_emul_vae.emulate(monkeypatch)
    a = _vae("batch2", micro_batch_size=1).decode(latents("batch2"), num_frames=17)
    b = _vae("batch2", micro_batch_size=None).decode(latents("batch2"), num_frames=17)
    assert torch.allclose(a, b, rtol=1e-5, atol=1e-5)


def test_opensora_vae_state_dict_layout_matches_reference():
    if not ref_loader.available():
        pytest.skip("reference checkout not present")
    from oracle.opensora_vae_ref import build_opensora_vae

    ref = build_opensora_vae(NARROW)
    ours = VideoAutoencoderPipeline(spatial_block_out_channels=NARROW)
    rs = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    os_ = {k: tuple(v.shape) for k, v in ours.state_dict().items()}
    # temporal part and the buffers: the reference's own modules, encoder side dropped
    want_t = {k: s for k, s in rs.items() if not k.startswith("spatial_vae.") and
              not k.startswith(("temporal_vae.encoder.", "temporal_vae.quant_conv."))}
    assert want_t == {k: s for k, s in os_.items() if not k.startswith("spatial_vae.")}
    # spatial part: the restated diffusers AutoencoderKL (decoder half) of oracle/sd_vae_ref.py
    assert {k: s for k, s in rs.items() if k.startswith("spatial_vae.")} == \
        {k: s for k, s in os_.items() if k.startswith("spatial_vae.")}
    ours.load_state_dict(weights(ref.state_dict(), "one_chunk"))  # the full reference dict: encoder keys dropped
    ref.load_state_dict({**ref.state_dict(), **ours.state_dict()}, strict=True)
    for k, v in ours.state_dict().items():
        assert torch.equal(ref.state_dict()[k], v)


def test_opensora_vae_released_spatial_keys():
    """The released image decoder has diffusers' key names for the SDXL VAE (block_out_channels 128, 256, 512, 512)."""
    keys = set(VideoAutoencoderPipeline().state_dict())
    p = "spatial_vae.module."
    for k in ("post_quant_conv.weight", "decoder.conv_in.weight", "decoder.mid_block.resnets.1.conv2.bias",
              "decoder.mid_block.attentions.0.group_norm.weight", "decoder.mid_block.attentions.0.to_out.0.weight",
              "decoder.up_blocks.2.resnets.0.conv_shortcut.weight", "decoder.up_blocks.3.resnets.0.conv_shortcut.bias",
              "decoder.up_blocks.2.upsamplers.0.conv.weight", "decoder.conv_norm_out.bias", "decoder.conv_out.weight"):
        assert p + k in keys, k
    assert not any(k.startswith(p + "decoder.up_blocks.3.upsamplers") for k in keys)
    assert not any(k.startswith(p + "decoder.up_blocks.0.resnets.0.conv_shortcut") for k in keys)
    assert {"scale", "shift", "temporal_vae.decoder.conv_out.conv.weight", "temporal_vae.decoder.conv_blocks.2.conv.bias"} <= keys
    assert not any(k.startswith("temporal_vae.decoder.conv_blocks.0.") for k in keys)  # nn.Identity level
    n = sum(v.numel() for k, v in VideoAutoencoderPipeline().state_dict().items() if k.startswith("temporal_vae."))
    assert 150e6 < n < 180e6


def _snapshot(tmp_path, name="one_chunk", drop=None):
    from safetensors.torch import save_file

    src = VideoAutoencoderPipeline(spatial_block_out_channels=NARROW)
    sd = weights(src.state_dict(), name)
    sd["scale"] = torch.tensor([1.5, 2.0, 2.5, 3.0]).view(1, 4, 1, 1, 1)  # checkpoint values load over the released ones
    full = {**sd, "temporal_vae.encoder.conv_in.conv.weight": torch.zeros(2), "temporal_vae.quant_conv.conv.bias": torch.zeros(8),
            "spatial_vae.module.encoder.conv_in.weight": torch.zeros(3), "spatial_vae.module.quant_conv.weight": torch.zeros(4)}
    if drop:
        full.pop(drop)
    d = tmp_path / "vae"
    d.mkdir()
    save_file({k: v.contiguous() for k, v in full.items()}, str(d / "model.safetensors"))
    return d, sd


def test_opensora_vae_from_pretrained_local_snapshot(tmp_path):
    d, sd = _snapshot(tmp_path)
    vae = VideoAutoencoderPipeline.from_pretrained(str(d), spatial_block_out_channels=NARROW)
    for k in ("scale", "temporal_vae.decoder.conv1.conv.weight", "spatial_vae.module.decoder.mid_block.attentions.0.to_q.bias"):
        assert torch.equal(vae.state_dict()[k], sd[k])
    assert vae.spatial_vae.micro_batch_size == 4 and vae.micro_z_frame_size == 5


def test_opensora_vae_from_pretrained_missing_decoder_key_raises(tmp_path):
    d, _ = _snapshot(tmp_path, drop="spatial_vae.module.decoder.conv_out.bias")
    with pytest.raises(RuntimeError, match="conv_out"):
        VideoAutoencoderPipeline.from_pretrained(str(d), spatial_block_out_channels=NARROW)
    with pytest.raises(FileNotFoundError):
        VideoAutoencoderPipeline.from_pretrained(str(tmp_path / "missing"))


def test_opensora_vae_rejections():
    with pytest.raises(NotImplementedError, match="encoder"):
        VideoAutoencoderPipeline(spatial_block_out_channels=NARROW).encode(torch.zeros(1, 3, 1, 8, 8))
    with pytest.raises(ValueError, match="spatial_block_out_channels"):
        VideoAutoencoderPipeline(spatial_block_out_channels=(96, 128, 256, 512))


# ---- the pipeline ----
class _StubScheduler:
    """Stands in for RFLOW.sample: returns fixed latents of the requested shape (the denoiser is not under test here)."""

    def sample(self, model, z, margs, y_null, dev, mask=None, progress=True):
        g = torch.Generator().manual_seed(7)
        return torch.randn(z.shape, generator=g).to(z.dtype)


class _StubTransformer(torch.nn.Module):
    in_channels = 4
    parallel_manager = None
    config = type("C", (), dict(model_max_length=4, caption_channels=8))()
    y_embedder = type("Y", (), dict(y_embedding=torch.zeros(4, 8)))()

    def reset_pab_state(self):
        pass


def _pipeline(vae, **kw):
    """An OpenSoraPipeline built without a GPU around a stub denoiser: only the decode stage is under test."""
    from videosys_b200.pipelines.open_sora import pipeline_open_sora as P

    pipe = P.OpenSoraPipeline.__new__(P.OpenSoraPipeline)
    pipe._config = P.OpenSoraConfig(num_sampling_steps=2, **({} if vae is None else dict(vae=vae)), **kw)
    pipe._device = torch.device("cpu")
    pipe.transformer = _StubTransformer()
    pipe.scheduler = _StubScheduler()
    pipe._set_seed = lambda seed: seed
    pipe._P = P
    return pipe, P


def _generate(pipe, monkeypatch):
    # 17 frames at a 16 x 24 image size (patched into the size table) -> latents [1, 4, 5, 2, 3]
    monkeypatch.setitem(pipe._P._IMAGE_SIZE, ("144p", "9:16"), (16, 24))
    return pipe.generate("a prompt", resolution="144p", aspect_ratio="9:16", num_frames=17, seed=0, verbose=False).video


def _reference_tail(vae, samples, num_frames):
    """The reference's lines after the sampler (pipeline_open_sora.py:638-648), on the same decoder."""
    video = vae.decode(samples.to(torch.bfloat16), num_frames=num_frames)
    low, high = -1, 1
    video.clamp_(min=low, max=high)
    video.sub_(low).div_(max(high - low, 1e-5))
    return video.mul(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 4, 1).to("cpu", torch.uint8)


def test_opensora_generate_with_native_vae_instance_and_dir(monkeypatch, tmp_path):
    kernels_emul_vae.emulate(monkeypatch)
    vae = _vae("one_chunk")
    pipe, _ = _pipeline(vae)
    pipe.vae = pipe._load_vae()
    assert pipe.vae is vae and vae.dtype == torch.bfloat16
    video = _generate(pipe, monkeypatch)
    assert video.dtype == torch.uint8 and tuple(video.shape) == (1, 17, 16, 24, 3)
    samples = _StubScheduler().sample(None, torch.zeros(1, 4, 5, 2, 3, dtype=torch.bfloat16), None, None, None)
    assert torch.equal(video, _reference_tail(vae, samples, 17))
    assert int(video.max()) > int(video.min())

    d, _ = _snapshot(tmp_path)
    pipe, _ = _pipeline(str(tmp_path), tiling_size=3)  # a snapshot root with a vae/ folder
    orig = VideoAutoencoderPipeline.from_pretrained.__func__
    monkeypatch.setattr(VideoAutoencoderPipeline, "from_pretrained", classmethod(
        lambda cls, path, subfolder=None, **k: orig(cls, path, subfolder, spatial_block_out_channels=NARROW, **k)))
    pipe.vae = pipe._load_vae()
    assert isinstance(pipe.vae, VideoAutoencoderPipeline) and pipe.vae.spatial_vae.micro_batch_size == 3


def test_opensora_generate_default_config_returns_latents(monkeypatch):
    kernels_emul_vae.emulate(monkeypatch)
    pipe, P = _pipeline(None)
    assert pipe._config.vae == "hpcai-tech/OpenSora-VAE-v1.2"
    pipe.vae = pipe._load_vae()
    assert pipe.vae is None
    lat = _generate(pipe, monkeypatch)
    want = _StubScheduler().sample(None, torch.zeros(1, 4, 5, 2, 3, dtype=torch.bfloat16), None, None, None)
    assert lat.dtype == torch.float32 and torch.equal(lat, want.float())


def test_opensora_generate_vae_decode_fn_takes_precedence(monkeypatch):
    kernels_emul_vae.emulate(monkeypatch)
    calls = []
    pipe, _ = _pipeline(_vae("image"), vae_decode_fn=lambda s, nf: calls.append((tuple(s.shape), nf)) or "decoded")
    pipe.vae = pipe._load_vae()
    assert pipe.vae is not None
    assert _generate(pipe, monkeypatch) == "decoded" and calls == [((1, 4, 5, 2, 3), 17)]
