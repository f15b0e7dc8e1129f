"""OpenSora v1.2 VAE decoder on the H100: the new kernel modes element by element against float64 (the rule of
tests/vae_fp64.py) -- GroupNorm + F.silu (act = 2) and the 4-channel causal conv_out with zero context frames --, the
depth-to-time shuffle bit for bit; the whole decoder against the reference's fp32 outputs within 1.25x of the eager
16-bit chain's own error; repeated decodes identical; one ``generate`` through the public engine with the native VAE."""
import os

import pytest
import torch

from oracle.gen_golden_opensora_vae import CASES, NARROW, latents, sample_index, weights
from tests import kernels_emul_vae as EV
from tests import vae_fp64 as V
from videosys_b200 import kernels
from videosys_b200.models.autoencoders import VideoAutoencoderPipeline

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _act(*shape, dtype, seed, offset=0.3):
    """Decoder-like activations, channels last: every third channel post-SiLU, a DC offset, four channels x 20."""
    z = torch.randn(*shape, generator=_gen(seed))
    z[..., ::3] = torch.nn.functional.silu(2 * z[..., ::3])
    z = z + offset
    z[..., :4] *= 20
    return z.to(dtype).to(DEV)


def _rand(*shape, dtype, scale=1.0, offset=0.0, seed=0):
    return (offset + scale * torch.randn(*shape, generator=_gen(seed))).to(dtype).to(DEV)


def silu_chain(n):
    """r(silu(n)) of F.silu: n / (1 + expf(-n)) in fp32, rounded once.  Where a legal input is below -80, expf(-n)
    overflows fp32 and the result may be anything down to zero (as in torch's own fp32 silu)."""
    fp32_range = torch.where(n.lo < -80, torch.full_like(n.v, 2.0**-100), torch.zeros_like(n.v))
    return n.step(V.silu64, eps=6 * V.U32 * V.silu64(n.v).abs() + fp32_range, turn=V.SILU_TURN)


def _nan_sentinels_intact(what, buf, t0, t1):
    outside = torch.cat([buf[:, :t0], buf[:, t1:]], 1)
    assert bool(torch.isnan(outside.float()).all()), f"{what}: wrote outside frames {t0}..{t1 - 1}"


# ---- GroupNorm + F.silu ----
GN_CASES = {"512ch_90x160_t2": (1, 2, 90, 160, 512), "128ch_180x1280_t1": (1, 1, 180, 1280, 128), "64ch_5x7_b2": (2, 3, 5, 7, 64)}


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("name", list(GN_CASES))
def test_vae_groupnorm_silu_fp64(name, eps, dtype):
    B, T, H, W, C = GN_CASES[name]
    x = _act(B, T, H, W, C, dtype=dtype, seed=1)
    gamma, beta = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=2), _rand(C, dtype=dtype, scale=0.1, seed=3)
    stats = kernels.vae_groupnorm_stats(x, 32, eps)
    buf = torch.full((B, T + 3, H, W, C), float("nan"), dtype=dtype, device=DEV)
    kernels.vae_groupnorm_act(x, stats, gamma, beta, out=buf, t_off=2, act=2)
    _nan_sentinels_intact("groupnorm_silu", buf, 2, 2 + T)
    V.assert_legal(f"groupnorm_silu {name} eps={eps} {dtype}", buf[:, 2:2 + T], silu_chain(V.gn_affine_chain(x, stats, gamma, beta)))
    again = kernels.vae_groupnorm_act(x, kernels.vae_groupnorm_stats(x, 32, eps), gamma, beta, act=2)
    assert torch.equal(again, buf[:, 2:2 + T])


# ---- the temporal decoder's conv_out: Cout = 4, zero context frames ----
CONV_CASES = {"128to4_90x160_t3": (1, 3, 90, 160, 128), "128to4_13x21_b2_t5": (2, 5, 13, 21, 128), "512to4_5x7": (1, 2, 5, 7, 512)}


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", list(CONV_CASES))
def test_vae_conv3d_cout4_zero_context_fp64(name, dtype):
    B, T, H, W, Cin = CONV_CASES[name]
    x = _act(B, T + 2, H, W, Cin, dtype=dtype, seed=4)
    x[:, :2] = 0  # CausalConv3d's F.pad(mode="constant") context
    w = _rand(4, Cin, 3, 3, 3, dtype=dtype, scale=(Cin * 27) ** -0.5, seed=5)
    wp = kernels.pack_conv_weight(w)
    for bias in (_rand(4, dtype=dtype, scale=0.1, seed=6), torch.zeros(4, dtype=dtype, device=DEV)):
        got = kernels.vae_conv3d(x, wp, bias, 4, 3)
        assert got.shape == (B, T, H, W, 4)
        V.assert_legal(f"conv3d Cout=4 {name} {dtype} bias={bool(bias.any())}", got, V.conv_chain(x, w, bias))


# ---- depth to time ----
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("B,T,H,W,C", [(1, 5, 90, 160, 512), (2, 3, 5, 7, 256), (1, 1, 1, 1, 8)])
def test_vae_depth_to_time_bit_exact(B, T, H, W, C, dtype):
    x = _act(B, T, H, W, 2 * C, dtype=dtype, seed=7)
    want = EV.vae_depth_to_time(x)  # the reference's einops rearrange
    V.assert_bit_exact(f"depth_to_time B={B} T={T} {H}x{W} C={C} {dtype}", kernels.vae_depth_to_time(x), want)
    buf = torch.full((B, 2 * T + 3, H, W, C), float("nan"), dtype=dtype, device=DEV)
    kernels.vae_depth_to_time(x, out=buf, t_off=2)
    _nan_sentinels_intact("depth_to_time", buf, 2, 2 + 2 * T)
    V.assert_bit_exact(f"depth_to_time t_off=2 {dtype}", buf[:, 2:2 + 2 * T], want)


# ---- the whole decoder ----
@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", "opensora_vae.pt"))


def _vae(name, dtype=torch.bfloat16):
    vae = VideoAutoencoderPipeline(spatial_block_out_channels=CASES[name][0])
    vae.load_state_dict(weights(vae.state_dict(), name))
    return vae.to(dtype).to(DEV).eval()


def _eager(monkeypatch, vae, z, nf):
    """The eager torch / cuDNN decoder: the same module on the kernels' stand-ins."""
    with monkeypatch.context() as m:
        for n, f in EV.stand_ins().items():
            m.setattr(kernels, n, f)
        return vae.decode(z, num_frames=nf)


@pytest.mark.parametrize("name", list(CASES))
def test_opensora_vae_decode_golden_within_eager16_error(monkeypatch, gold, name):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    vae = _vae(name)
    nf = CASES[name][2]
    z = latents(name).to(DEV)
    n0 = kernels.launch_count()
    ours = vae.decode(z, num_frames=nf)
    assert kernels.launch_count() - n0 > 50
    assert list(ours.shape) == gold[f"{name}.shape"]
    assert torch.equal(ours, vae.decode(z, num_frames=nf)), "two decodes differ"
    eager = _eager(monkeypatch, vae, z, nf)
    want = gold[f"{name}.fp32"].double()
    idx = sample_index(ours.numel(), name).to(DEV) if ours.numel() > want.numel() else torch.arange(ours.numel(), device=DEV)
    e_ours = float((ours.flatten()[idx].double().cpu() - want).norm())
    e_eager = float((eager.flatten()[idx].double().cpu() - want).norm())
    print(f"[decode {name}] |ours - ref| = {e_ours:.4g}, |eager16 - ref| = {e_eager:.4g}, ratio {e_ours / e_eager:.3f}")
    assert e_ours <= 1.25 * e_eager


def test_opensora_generate_with_native_vae():
    from videosys_b200 import OpenSoraConfig, VideoSysEngine
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3Config

    vae = VideoAutoencoderPipeline(spatial_block_out_channels=NARROW)
    vae.load_state_dict(weights(vae.state_dict(), "one_chunk"))
    tcfg = STDiT3Config(hidden_size=288, num_heads=4, depth=2, caption_channels=64, model_max_length=24)
    eng = VideoSysEngine(OpenSoraConfig(num_sampling_steps=2, transformer_config=tcfg, vae=vae))
    try:
        assert eng.driver_worker.vae is vae and vae.dtype == torch.bfloat16
        out = eng.generate("Sunset over the sea.", resolution="144p", aspect_ratio="9:16", num_frames=17, seed=0, verbose=False).video
    finally:
        eng.shutdown()
    assert out.dtype == torch.uint8 and tuple(out.shape) == (1, 17, 144, 256, 3)
    assert int(out.max()) > int(out.min())
