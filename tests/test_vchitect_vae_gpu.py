"""Vchitect-2.0 VAE decode on the H100: the golden decodes against the restated reference's fp32 outputs within 1.25x of
the eager 16-bit chain's own error, and ``generate`` end to end through the public engine with the native VAE."""
import os

import pytest
import torch

from oracle import gen_golden_latte_vae as G
from oracle.gen_golden_opensora_vae import NARROW, weights
from tests import kernels_emul_vae_time as EV
from videosys_b200 import kernels
from videosys_b200.models.autoencoders import AutoencoderKL

pytestmark = pytest.mark.gpu
DEV = "cuda"
SMALL = dict(sample_size=8, patch_size=2, in_channels=16, num_layers=2, attention_head_dim=64, num_attention_heads=2,
             joint_attention_dim=48, caption_projection_dim=128, pooled_projection_dim=40, out_channels=16, pos_embed_max_size=12)


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", "vchitect_vae.pt"))


def _vae(name, widths=None):
    vae = AutoencoderKL(block_out_channels=widths or G.VCHITECT_CASES[name][0], latent_channels=16, use_post_quant_conv=False,
                        scaling_factor=G.VCH_SCALE, shift_factor=G.VCH_SHIFT)
    vae.load_state_dict(weights(vae.state_dict(), "vchitect/" + name))
    return vae


def _decoded(vae, z):
    """The pipeline's decode tail up to the post-processing (pipeline_vchitect.py:980-983)."""
    from videosys_b200.pipelines._common import decode_image_frames

    return decode_image_frames(vae, ((z / vae.config.scaling_factor) + vae.config.shift_factor)[0])


@pytest.mark.parametrize("name", list(G.VCHITECT_CASES))
def test_vchitect_vae_decode_golden_within_eager16_error(monkeypatch, gold, name):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    vae = _vae(name).to(torch.bfloat16).to(DEV).eval()
    z = G.latents("vchitect/" + name, G.VCHITECT_CASES[name][1]).to(torch.bfloat16).to(DEV)
    ours = _decoded(vae, z)
    assert list(ours.shape) == gold[f"{name}.shape"]
    assert torch.equal(ours, _decoded(vae, z)), "two decodes differ"
    with monkeypatch.context() as m:
        for n, f in EV.stand_ins().items():
            m.setattr(kernels, n, f)
        eager = _decoded(vae, z)
    want = gold[f"{name}.fp32"].double()
    idx = G.sample_index(ours.numel(), name).to(DEV) if ours.numel() > want.numel() else torch.arange(ours.numel(), device=DEV)
    e_ours = float((ours.flatten()[idx].double().cpu() - want).norm())
    e_eager = float((eager.flatten()[idx].double().cpu() - want).norm())
    print(f"[vchitect decode {name}] |ours - ref| = {e_ours:.4g}, |eager16 - ref| = {e_eager:.4g}, ratio {e_ours / e_eager:.3f}")
    assert e_ours <= 1.25 * e_eager


def test_vchitect_generate_with_native_vae():
    from videosys_b200 import VchitectConfig, VideoSysEngine

    vae = _vae("narrow", NARROW)
    eng = VideoSysEngine(VchitectConfig(transformer_config=SMALL, vae=vae))
    try:
        assert eng.driver_worker.vae is vae and vae.dtype == torch.bfloat16
        out = eng.generate("Sunset over the sea.", num_inference_steps=2, seed=0, frames=4, height=96, width=128,
                           output_type="np").video
    finally:
        eng.shutdown()
    assert len(out) == 1 and len(out[0]) == 4
    assert out[0][0].shape == (96, 128, 3) and str(out[0][0].dtype) == "float32"
    assert 0.0 <= float(out[0][0].min()) < float(out[0][0].max()) <= 1.0
