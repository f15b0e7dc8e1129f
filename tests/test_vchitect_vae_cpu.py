"""Vchitect-2.0 VAE decode: the image VAE with 16 latent channels, no post_quant_conv and a shift_factor, and
VchitectXLPipeline's decode tail and per-frame post-processing, on the torch stand-ins of the kernels, fp32, against
the restated reference in tests/golden/vchitect_vae.pt (oracle/gen_golden_latte_vae.py); the state-dict layout;
snapshot loading; the frame batching; and ``generate`` around a stub denoiser."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import gen_golden_latte_vae as G
from oracle.gen_golden_opensora_vae import NARROW, weights
from tests import kernels_emul_vae_time
from videosys_b200.models.autoencoders import AutoencoderKL
from videosys_b200.pipelines import _common

_CFG = dict(_class_name="AutoencoderKL", block_out_channels=list(NARROW), latent_channels=16, layers_per_block=2,
            scaling_factor=G.VCH_SCALE, shift_factor=G.VCH_SHIFT, use_quant_conv=False, use_post_quant_conv=False)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "vchitect_vae.pt"))


def _vae(name):
    vae = AutoencoderKL.from_config({**_CFG, "block_out_channels": G.VCHITECT_CASES[name][0]}).eval()
    vae.load_state_dict(weights(vae.state_dict(), "vchitect/" + name))
    return vae


class _StubTransformer(torch.nn.Module):
    config = type("C", (), dict(in_channels=16, joint_attention_dim=8, pooled_projection_dim=8))()
    parallel_manager = None

    def reset_pab_state(self):
        pass

    def forward(self, x, **kw):
        return (0.1 * x,)


def _pipeline(vae, **kw):
    from videosys_b200.pipelines.vchitect import pipeline_vchitect as P

    pipe = P.VchitectXLPipeline.__new__(P.VchitectXLPipeline)
    pipe._config = P.VchitectConfig(vae=vae, **kw)
    pipe._device, pipe._dtype = torch.device("cpu"), torch.float32
    pipe.transformer = _StubTransformer()
    pipe.scheduler = P.FlowMatchEulerDiscreteScheduler(shift=3.0)
    pipe.vae = pipe._load_vae()
    return pipe


def _generate(pipe, **kw):
    e = torch.zeros(1, 4, 8)
    p = torch.zeros(1, 8)
    return pipe.generate(prompt_embeds=e, negative_prompt_embeds=e, pooled_prompt_embeds=p, negative_pooled_prompt_embeds=p,
                         num_inference_steps=2, seed=0, frames=3, height=16, width=24, **kw).video


@pytest.mark.parametrize("name", list(G.VCHITECT_CASES))
def test_vchitect_vae_decode_vs_reference_golden(monkeypatch, gold, name):
    kernels_emul_vae_time.emulate(monkeypatch)
    pipe = _pipeline(_vae(name))
    z = G.latents("vchitect/" + name, G.VCHITECT_CASES[name][1])
    video = pipe.decode_latents_to_video(z, "pt")
    assert len(video) == 1 and len(video[0]) == z.shape[1]
    out = torch.stack(video[0]) * 2 - 1  # undo the post-processing's (x / 2 + 0.5), exact in fp32 up to the clamp
    want = gold[f"{name}.fp32"]
    assert list(out.shape) == gold[f"{name}.shape"]
    flat = out.flatten()
    got = flat[G.sample_index(flat.numel(), name)] if flat.numel() > want.numel() else flat
    inside = want.abs() < 1  # the clamp to [0, 1] of the post-processing
    assert torch.allclose(got[inside], want[inside], rtol=1e-4, atol=1e-4), (got - want)[inside].abs().max()
    assert torch.equal(got[~inside], want[~inside].clamp(-1, 1))


def test_vchitect_vae_frames_per_pass_do_not_change_the_result(monkeypatch):
    kernels_emul_vae_time.emulate(monkeypatch)
    pipe = _pipeline(_vae("narrow"))
    z = G.latents("vchitect/narrow", G.VCHITECT_CASES["narrow"][1])
    a = pipe.decode_latents_to_video(z, "pt")
    monkeypatch.setattr(_common, "VAE_FRAMES_PER_PASS", 1)
    b = pipe.decode_latents_to_video(z, "pt")
    assert all(torch.allclose(x, y, rtol=1e-5, atol=1e-5) for x, y in zip(a[0], b[0]))


def test_vchitect_vae_state_dict_layout_matches_reference():
    ref = G.VchitectVAE(NARROW)
    assert {k: tuple(v.shape) for k, v in ref.state_dict().items()} == {k: tuple(v.shape) for k, v in _vae("narrow").state_dict().items()}


def _snapshot(tmp_path, drop=None):
    from safetensors.torch import save_file

    sd = {**_vae("narrow").state_dict(), "encoder.conv_in.weight": torch.zeros(2)}
    if drop:
        sd.pop(drop)
    d = tmp_path / "vae"
    d.mkdir(parents=True)
    (d / "config.json").write_text(json.dumps(_CFG))
    save_file({k: v.contiguous() for k, v in sd.items()}, str(d / "diffusion_pytorch_model.safetensors"))
    return tmp_path


def test_vchitect_vae_from_pretrained_local_snapshot(tmp_path):
    vae = AutoencoderKL.from_pretrained(str(_snapshot(tmp_path)))
    assert vae.post_quant_conv is None and vae.config.latent_channels == 16 and vae.config.shift_factor == G.VCH_SHIFT
    for k, v in _vae("narrow").state_dict().items():
        assert torch.equal(vae.state_dict()[k], v)
    with pytest.raises(RuntimeError, match="conv_norm_out"):
        AutoencoderKL.from_pretrained(str(_snapshot(tmp_path / "m", drop="decoder.conv_norm_out.weight")))


def test_vchitect_generate_with_native_vae(monkeypatch, tmp_path):
    kernels_emul_vae_time.emulate(monkeypatch)
    pipe = _pipeline(_vae("narrow"))
    for ot in ("np", "pil", "pt"):
        video = _generate(pipe, output_type=ot)
        assert len(video) == 1 and len(video[0]) == 3
        if ot == "np":
            assert video[0][0].shape == (16, 24, 3) and video[0][0].dtype == np.float32
            arr = np.stack(video[0])
        elif ot == "pil":
            assert video[0][0].size == (24, 16)
            assert np.array_equal(np.asarray(video[0][1]), (arr[1] * 255).round().astype("uint8"))
        else:
            assert tuple(video[0][2].shape) == (3, 16, 24)
    pipe = _pipeline(str(_snapshot(tmp_path)))
    assert isinstance(pipe.vae, AutoencoderKL) and pipe.vae.config.latent_channels == 16


def test_vchitect_generate_vae_decode_fn_takes_precedence_and_default_returns_latents(monkeypatch):
    kernels_emul_vae_time.emulate(monkeypatch)
    calls = []
    pipe = _pipeline(_vae("narrow"), vae_decode_fn=lambda s: calls.append(tuple(s.shape)) or "decoded")
    assert _generate(pipe) == "decoded" and calls == [(1, 3, 16, 2, 3)]
    pipe = _pipeline(None)
    assert pipe.vae is None
    lat = _generate(pipe)
    assert lat.dtype == torch.float32 and tuple(lat.shape) == (1, 3, 16, 2, 3)
