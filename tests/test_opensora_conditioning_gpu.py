"""OpenSora v1.2 conditioning end to end on the H100: ``generate(refs=<png>, ms="0")`` and ``generate(loop=2)`` through
the public engine with a small STDiT3 and the narrow native VAE; the conditioning latents the sampler receives against
the eager 16-bit encoder chain (tests/kernels_emul_vae_down.py) on the same inputs and seed."""
import pytest
import torch

from oracle.gen_golden_opensora_vae import NARROW, weights
from tests import kernels_emul_vae_down as ED
from videosys_b200 import kernels
from videosys_b200.models.autoencoders import OpenSoraVAEEncoder, VideoAutoencoderPipeline

pytestmark = pytest.mark.gpu


def _engine():
    from videosys_b200 import OpenSoraConfig, VideoSysEngine
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3Config

    vae = VideoAutoencoderPipeline(spatial_block_out_channels=NARROW)
    vae.load_state_dict(weights(vae.state_dict(), "one_chunk"))
    enc = OpenSoraVAEEncoder(spatial_block_out_channels=NARROW)
    enc.load_state_dict(weights(enc.state_dict(), "one_chunk"))
    tcfg = STDiT3Config(hidden_size=288, num_heads=4, depth=2, caption_channels=64, model_max_length=24)
    return VideoSysEngine(OpenSoraConfig(num_sampling_steps=2, transformer_config=tcfg, vae=vae, vae_encoder=enc)), enc


def _record(monkeypatch, pipe):
    calls = []
    orig = pipe.scheduler.sample

    def sample(model, z, *a, mask=None, **k):
        calls.append((z.clone(), mask.clone()))
        return orig(model, z, *a, mask=mask, **k)

    monkeypatch.setattr(pipe.scheduler, "sample", sample)
    return calls


def _eager_encode(monkeypatch, enc, x, seed_fn):
    with monkeypatch.context() as m:
        for n, f in ED.stand_ins().items():
            m.setattr(kernels, n, f)
        seed_fn()
        return enc.encode(x.to(enc.device, enc.dtype))


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_generate_image_ref_and_loop(monkeypatch, tmp_path):
    from PIL import Image

    from videosys_b200.pipelines.open_sora.conditioning import load_image

    g = torch.Generator().manual_seed(0)
    png = str(tmp_path / "ref.png")
    Image.fromarray(torch.randint(0, 256, (300, 500, 3), generator=g, dtype=torch.uint8).numpy()).save(png)
    eng, enc = _engine()
    try:
        pipe = eng.driver_worker
        calls = _record(monkeypatch, pipe)
        n0 = kernels.launch_count()
        out = eng.generate("Sunset over the sea.", resolution="144p", aspect_ratio="9:16", num_frames=17, seed=0,
                           refs=png, ms="0", verbose=False).video
        assert kernels.launch_count() - n0 > 100
        assert out.dtype == torch.uint8 and tuple(out.shape) == (1, 17, 144, 256, 3)
        (z, mask), = calls
        assert mask.tolist() == [[0.0, 1.0, 1.0, 1.0, 1.0]]
        ref = _eager_encode(monkeypatch, enc, load_image(png, (144, 256))[None], lambda: pipe._set_seed(0))[0]
        rel = _rel(z[0, :, 0], ref[:, 0])
        print(f"[refs] conditioning frame native vs eager16: rel L2 {rel:.3e}")
        assert rel < 5e-2

        calls.clear()
        decoded = []
        orig_dec = pipe.vae.decode
        monkeypatch.setattr(pipe.vae, "decode", lambda z, num_frames=None: decoded.append(orig_dec(z, num_frames)) or decoded[-1])
        out = eng.generate("Sunset over the sea.", resolution="144p", aspect_ratio="9:16", num_frames=34, seed=0, loop=2,
                           verbose=False).video
        assert tuple(out.shape) == (1, 34 + 17, 144, 256, 3)
        (_, m0), (_, m1) = calls
        assert bool((m0 == 1).all()) and bool((m1[0, :5] == 0).all()) and bool((m1[0, 5:] == 1).all())
        # the first clip re-encoded (the RNG state at the re-encode: after seed, z of loop 0 and its sampling) --
        # compare the posterior means, which do not depend on it
        with monkeypatch.context() as m:
            m.setattr(torch, "randn", lambda *s, **kw: torch.zeros(*s, **{k: v for k, v in kw.items() if k != "generator"}))
            mean_native = enc.encode(decoded[0])
            mean_eager = _eager_encode(monkeypatch, enc, decoded[0], lambda: None)
        rel = _rel(mean_native, mean_eager)
        print(f"[loop] re-encoded first clip means native vs eager16: rel L2 {rel:.3e}")
        assert rel < 5e-2
    finally:
        eng.shutdown()
