"""Latte VAE decode on the H100: the golden decodes (temporal decoder, chunk straddling two samples, image path, image
VAE, released widths) against the restated reference's fp32 outputs within 1.25x of the eager 16-bit chain's own error;
one decode at Latte's real shape against the eager chain; ``generate`` end to end through the public engine."""
import os

import pytest
import torch

from oracle import gen_golden_latte_vae as G
from oracle.gen_golden_opensora_vae import NARROW, RELEASED, weights
from tests import kernels_emul_vae_time as EV
from videosys_b200 import kernels
from videosys_b200.models.autoencoders import AutoencoderKL, AutoencoderKLTemporalDecoder

pytestmark = pytest.mark.gpu
DEV = "cuda"
SMALL = dict(num_attention_heads=4, attention_head_dim=72, in_channels=4, out_channels=8, num_layers=2, sample_size=16,
             caption_channels=64, video_length=6)


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", "latte_vae.pt"))


def _vae(name, dtype=torch.float16):
    kind, widths, _ = G.LATTE_CASES[name]
    vae = (AutoencoderKLTemporalDecoder if kind == "temporal" else AutoencoderKL)(block_out_channels=widths)
    vae.load_state_dict(weights(vae.state_dict(), "latte/" + name))
    return vae.to(dtype).to(DEV).eval()


def _pipeline(vae):
    from videosys_b200.pipelines.latte import pipeline_latte as P

    pipe = P.LattePipeline.__new__(P.LattePipeline)
    pipe._config, pipe._device, pipe._dtype, pipe.vae = P.LatteConfig(vae=vae), torch.device(DEV), torch.float16, vae
    return pipe


def _decode(pipe, z):
    return pipe.decode_latents_image(z) if z.shape[2] == 1 else pipe.decode_video(z)


def _eager(monkeypatch, fn):
    """fn() on the kernels' stand-ins: the eager torch / cuDNN chain of the same modules."""
    with monkeypatch.context() as m:
        for n, f in EV.stand_ins().items():
            m.setattr(kernels, n, f)
        return fn()


@pytest.mark.parametrize("name", list(G.LATTE_CASES))
def test_latte_vae_decode_golden_within_eager16_error(monkeypatch, gold, name):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    pipe = _pipeline(_vae(name))
    z = G.latents("latte/" + name, G.LATTE_CASES[name][2]).to(torch.float16).to(DEV)
    n0 = kernels.launch_count()
    ours = _decode(pipe, z)
    assert kernels.launch_count() - n0 > 30
    assert list(ours.shape) == gold[f"{name}.shape"]
    assert torch.equal(ours, _decode(pipe, z)), "two decodes differ"
    eager = _eager(monkeypatch, lambda: _decode(pipe, z))
    want = gold[f"{name}.fp32"].double()
    idx = G.sample_index(ours.numel(), name).to(DEV) if ours.numel() > want.numel() else torch.arange(ours.numel(), device=DEV)
    e_ours = float((ours.flatten()[idx].double().cpu() - want).norm())
    e_eager = float((eager.flatten()[idx].double().cpu() - want).norm())
    print(f"[latte decode {name}] |ours - ref| = {e_ours:.4g}, |eager16 - ref| = {e_eager:.4g}, ratio {e_ours / e_eager:.3f}")
    assert e_ours <= 1.25 * e_eager


def test_latte_vae_real_shape_against_eager(monkeypatch):
    """Latents [1, 4, 16, 64, 64] (16 frames at 512 x 512), released widths, fp16."""
    vae = AutoencoderKLTemporalDecoder(block_out_channels=RELEASED)
    vae.load_state_dict(weights(vae.state_dict(), "latte/real"))
    pipe = _pipeline(vae.half().to(DEV).eval())
    z = torch.randn(1, 4, 16, 64, 64, generator=torch.Generator().manual_seed(0)).half().to(DEV)
    ours = pipe.decode_video(z)
    assert tuple(ours.shape) == (1, 16, 512, 512, 3) and bool(torch.isfinite(ours).all())
    eager = _eager(monkeypatch, lambda: pipe.decode_video(z))
    d = (ours.float() - eager.float()).abs()
    print(f"[latte real shape] |native - eager| on the [-1, 1] scale: max {float(d.max()):.4f}, mean {float(d.mean()):.3e}; "
          f"mean |eager| {float(eager.float().abs().mean()):.3f}")
    assert float(d.mean()) < 2e-2 * float(eager.float().abs().mean()) + 1e-3


def test_latte_generate_with_native_vae():
    from videosys_b200 import LatteConfig, VideoSysEngine

    vae = AutoencoderKLTemporalDecoder(block_out_channels=NARROW)
    vae.load_state_dict(weights(vae.state_dict(), "latte/temporal_16"))
    eng = VideoSysEngine(LatteConfig(transformer_config=SMALL, vae=vae))
    try:
        assert eng.driver_worker.vae is vae and vae.dtype == torch.float16
        out = eng.generate("Sunset over the sea.", num_inference_steps=2, seed=0, video_length=6, height=128, width=128).video
    finally:
        eng.shutdown()
    assert out.dtype == torch.uint8 and out.device.type == "cpu" and tuple(out.shape) == (1, 6, 128, 128, 3)
    assert int(out.max()) > int(out.min())
