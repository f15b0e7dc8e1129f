"""OpenSora v1.2 VAE encoder: the host logic (image micro-batches, 17-frame chunks, zero time padding in front, the zero
causal context and the strided convolutions' inputs, RGB / latent channel padding, the posterior's noise draws and
their order, (z - shift) / scale) on the torch stand-ins of the kernels (tests/kernels_emul_vae_down.py), fp32, against
the UNMODIFIED reference encode in tests/golden/opensora_vae_encode.pt (oracle/gen_golden_opensora_vae_encode.py) and
live when the reference checkout is present; the state-dict layout and snapshot loading of both halves."""
import os

import pytest
import torch

from oracle import ref_loader
from oracle.gen_golden_opensora_vae import NARROW, weights
from oracle.gen_golden_opensora_vae_encode import CASES, SEED, sample_index, videos
from tests import kernels_emul_vae_down
from videosys_b200.models.autoencoders import OpenSoraVAEEncoder, VideoAutoencoderPipeline


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "opensora_vae_encode.pt"))


def _enc(name, **kw):
    enc = OpenSoraVAEEncoder(spatial_block_out_channels=CASES[name][0], **kw).eval()
    enc.load_state_dict(weights(enc.state_dict(), name))
    return enc


def _zero_noise(monkeypatch):
    """torch.randn -> zeros: the posteriors' samples become their means."""
    monkeypatch.setattr(torch, "randn", lambda *s, **kw: torch.zeros(*s, **{k: v for k, v in kw.items() if k != "generator"}))


def _subset(y, name, want):
    flat = y.flatten()
    return flat[sample_index(flat.numel(), name)] if flat.numel() > want.numel() else flat


@pytest.mark.parametrize("name", list(CASES))
def test_opensora_vae_encode_vs_reference_golden(monkeypatch, gold, name):
    kernels_emul_vae_down.emulate(monkeypatch)
    enc = _enc(name)
    torch.manual_seed(SEED)
    z = enc.encode(videos(name))
    assert list(z.shape) == gold[f"{name}.shape"]
    want = gold[f"{name}.z"]
    got = _subset(z, name, want)
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-4), (got - want).abs().max()
    _zero_noise(monkeypatch)
    want = gold[f"{name}.mode"]
    got = _subset(enc.encode(videos(name)), name, want)
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-4), (got - want).abs().max()


def test_opensora_vae_encode_vs_live_reference(monkeypatch):
    """The reference's VideoAutoencoderPipeline.encode and temporal Encoder executed as written, same seed: every Gaussian
    draw is consumed in the same order and shape (a change of either moves z far off)."""
    if not ref_loader.available():
        pytest.skip("reference checkout not present")
    from oracle.sd_vae_encoder_ref import build_opensora_vae_full

    kernels_emul_vae_down.emulate(monkeypatch)
    ref = build_opensora_vae_full(NARROW)
    sd = weights(ref.state_dict(), "live")
    ref.load_state_dict(sd)
    enc = OpenSoraVAEEncoder(spatial_block_out_channels=NARROW, micro_batch_size=3).eval()
    enc.load_state_dict(sd)
    ref.spatial_vae.micro_batch_size = 3
    x = 2 * torch.rand(2, 3, 19, 16, 24, generator=torch.Generator().manual_seed(0)) - 1
    with torch.no_grad():
        torch.manual_seed(5)
        want = ref.encode(x)
        after_ref = torch.randn(4)
    torch.manual_seed(5)
    got = enc.encode(x)
    assert torch.equal(torch.randn(4), after_ref), "the encoder drew a different number of random values"
    assert got.shape == want.shape == (2, 4, 6, 2, 3)
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-4), (got - want).abs().max()


def test_opensora_vae_encoder_keys_are_the_reference_encoder_side():
    ours = {k: tuple(v.shape) for k, v in OpenSoraVAEEncoder(spatial_block_out_channels=NARROW).state_dict().items()}
    assert all(k.startswith(OpenSoraVAEEncoder._KEPT_PREFIXES) for k in ours)
    released = set(OpenSoraVAEEncoder().state_dict())
    p = "spatial_vae.module."
    for k in ("quant_conv.weight", "encoder.conv_in.weight", "encoder.down_blocks.0.downsamplers.0.conv.weight",
              "encoder.down_blocks.1.resnets.0.conv_shortcut.bias", "encoder.mid_block.attentions.0.to_q.weight",
              "encoder.conv_norm_out.bias", "encoder.conv_out.weight"):
        assert p + k in released, k
    assert not any(k.startswith(p + "encoder.down_blocks.3.downsamplers") for k in released)
    assert {"temporal_vae.encoder.conv_in.conv.weight", "temporal_vae.encoder.conv_blocks.1.conv.bias",
            "temporal_vae.encoder.conv2.conv.weight", "temporal_vae.quant_conv.conv.bias"} <= released
    assert not any(k.startswith("temporal_vae.encoder.conv_blocks.0.") for k in released)  # nn.Identity level
    if not ref_loader.available():
        return
    from oracle.sd_vae_encoder_ref import build_opensora_vae_full

    rs = {k: tuple(v.shape) for k, v in build_opensora_vae_full(NARROW).state_dict().items()}
    assert ours == {k: s for k, s in rs.items() if k.startswith(OpenSoraVAEEncoder._KEPT_PREFIXES)}
    # the two halves cover the checkpoint: every other key is the decoder's or a buffer
    dec = set(VideoAutoencoderPipeline(spatial_block_out_channels=NARROW).state_dict())
    assert set(rs) == set(ours) | dec


def _snapshot(tmp_path, drop=None):
    """model.safetensors with both halves (and scale / shift), as the released checkpoint has them."""
    from safetensors.torch import save_file

    enc = OpenSoraVAEEncoder(spatial_block_out_channels=NARROW)
    dec = VideoAutoencoderPipeline(spatial_block_out_channels=NARROW)
    full = {**weights(dec.state_dict(), "snap"), **weights(enc.state_dict(), "snap")}
    full["scale"] = torch.tensor([1.5, 2.0, 2.5, 3.0]).view(1, 4, 1, 1, 1)
    if drop:
        full.pop(drop)
    d = tmp_path / "vae"
    d.mkdir()
    save_file({k: v.contiguous() for k, v in full.items()}, str(d / "model.safetensors"))
    return d, full


def test_opensora_vae_encoder_from_pretrained_both_halves(tmp_path):
    d, full = _snapshot(tmp_path)
    enc = OpenSoraVAEEncoder.from_pretrained(str(d), spatial_block_out_channels=NARROW)
    dec = VideoAutoencoderPipeline.from_pretrained(str(d), spatial_block_out_channels=NARROW)
    for k, v in enc.state_dict().items():
        assert torch.equal(v, full[k]), k
    for k, v in dec.state_dict().items():
        assert torch.equal(v, full[k]), k
    assert torch.equal(enc.scale, full["scale"]) and torch.equal(enc.shift, dec.shift)
    assert enc.spatial_vae.micro_batch_size == 4 and enc.micro_frame_size == 17


def test_opensora_vae_encoder_missing_key_raises(tmp_path):
    d, _ = _snapshot(tmp_path, drop="spatial_vae.module.encoder.conv_out.bias")
    with pytest.raises(RuntimeError, match="conv_out"):
        OpenSoraVAEEncoder.from_pretrained(str(d), spatial_block_out_channels=NARROW)
    with pytest.raises(ValueError, match="spatial_block_out_channels"):
        OpenSoraVAEEncoder(spatial_block_out_channels=(96, 128, 256, 512))


def test_opensora_vae_encoder_needs_cuda_and_16_bits():
    """Without the stand-ins the encoder runs on the kernels only: a CPU input is refused, not run eagerly."""
    with pytest.raises(RuntimeError, match="CUDA"):
        OpenSoraVAEEncoder(spatial_block_out_channels=NARROW).encode(torch.zeros(1, 3, 1, 16, 16))
