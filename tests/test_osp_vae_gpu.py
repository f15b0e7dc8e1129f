"""Open-Sora-Plan causal-VAE decoder on the H100: each new kernel against eager torch laid out the way the reference calls
it (F.group_norm + x * torch.sigmoid(x), torch.bmm / softmax on the (b*t, c, h*w) views, F.interpolate trilinear) in bf16
and fp16 at released shapes, with the bit-equal fraction and the largest error in ulps reported; repeated launches
identical; the whole decoder against the reference's fp32 outputs within 1.25x of the eager 16-bit decoder's own error;
one ``generate`` with the native decoder."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle.gen_golden_osp_vae import CASES, apply_tiling, latents, sample_index, weights
from tests import kernels_emul_vae as EV
from videosys_b200 import kernels
from videosys_b200.models.autoencoders._common import frame_attention
from videosys_b200.models.autoencoders.autoencoder_kl_open_sora_plan import decoder_class

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]


def _ulps(got, want):
    g, w = got.float(), want.float()
    mag = torch.maximum(g.abs(), w.abs()).to(want.dtype)
    ulp = (torch.nextafter(mag, torch.full_like(mag, float("inf"))) - mag).float()
    return ((g - w).abs() / ulp).double()


def _report(what, got, want):
    u = _ulps(got, want)
    eq = float((got == want).float().mean())
    print(f"[{what}] bit-equal {100 * eq:.4f} %, max {float(u.max()):.0f} ulp")
    return eq, float(u.max())


@pytest.fixture
def no_tf32(monkeypatch):
    """fp32 references without TF32, restored afterwards for the tests that follow."""
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)


def _rand(*shape, dtype, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (scale * torch.randn(*shape, generator=g)).to(dtype).to(DEV)


# ---- GroupNorm (+ nonlinearity) ----
GN_SHAPES = {"512ch_60x80_t3": (3, 60, 80, 512), "128ch_480x640_t2": (2, 480, 640, 128)}


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("act", [True, False], ids=["act", "noact"])
@pytest.mark.parametrize("name", list(GN_SHAPES))
def test_vae_groupnorm_act_vs_eager(name, act, dtype):
    T, H, W, C = GN_SHAPES[name]
    x = _rand(1, T, H, W, C, dtype=dtype, scale=2.0, seed=1) + 0.5
    gamma, beta = _rand(C, dtype=dtype, scale=0.2, seed=2) + 1, _rand(C, dtype=dtype, scale=0.1, seed=3)
    n = F.group_norm(x.permute(0, 4, 1, 2, 3), 32, gamma, beta, 1e-6)
    want = (n * torch.sigmoid(n) if act else n).permute(0, 2, 3, 4, 1)
    stats = kernels.vae_groupnorm_stats(x, 32, 1e-6)
    buf = torch.empty(1, T + 2, H, W, C, dtype=dtype, device=DEV)
    got = kernels.vae_groupnorm_act(x, stats, gamma, beta, out=buf, t_off=2, act=act)[:, 2:]
    eq, ulp = _report(f"groupnorm_act {name} act={int(act)} {dtype}", got, want)
    again = torch.empty_like(buf)
    kernels.vae_groupnorm_act(x, kernels.vae_groupnorm_stats(x, 32, 1e-6), gamma, beta, out=again, t_off=2, act=act)
    assert torch.equal(again[:, 2:], got)
    # mean / rstd are summed in another order than torch's Welford; where their 16-bit rounding flips, a whole group moves
    # by an ulp of the normalised value
    assert eq >= 0.9 and ulp <= 8


# ---- attention ----
ATTN_SHAPES = {"fix_60x80_t1": (1, 60, 80, False), "attn3d_64x64_t2": (2, 64, 64, True)}


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("name", list(ATTN_SHAPES))
def test_vae_attention_vs_eager(name, dtype, no_tf32):
    T, H, W, mixed = ATTN_SHAPES[name]
    C = 512
    qkv = _rand(1, T, H, W, 3 * C, dtype=dtype, scale=1.5, seed=4)
    ours = frame_attention(qkv, C, mixed)
    eager = EV.eager_attention(qkv, C, mixed)
    ref = EV.eager_attention(qkv.float(), C, mixed).double()
    _report(f"attention {name} {dtype}", ours, eager)
    e_ours, e_eager = float((ours.double() - ref).norm()), float((eager.double() - ref).norm())
    print(f"[attention {name} {dtype}] |ours - fp32| = {e_ours:.4g}, |eager16 - fp32| = {e_eager:.4g}, ratio {e_ours / e_eager:.3f}")
    assert torch.equal(ours, frame_attention(qkv, C, mixed))
    assert e_ours <= 1.25 * e_eager


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("P", [4800, 4096, 15])
def test_vae_attn_softmax_vs_eager(P, dtype):
    Pp = -(-P // 8) * 8
    S = _rand(P, Pp, dtype=dtype, scale=8.0, seed=5)
    want = F.softmax(S[:, :P] * (512 ** -0.5), dim=-1)
    got = kernels.vae_attn_softmax_(S.clone(), P, 512 ** -0.5)
    eq, ulp = _report(f"attn_softmax P={P} {dtype}", got[:, :P], want)
    assert bool((got[:, P:] == 0).all())
    assert torch.equal(got, kernels.vae_attn_softmax_(S.clone(), P, 512 ** -0.5))
    assert eq >= 0.99 and ulp <= 1  # the row sum runs in another order than ATen's


# ---- linear up-sampler and the TimeUpsampleRes2x mix ----
LIN_SHAPES = {"spatial_time_256_120x160_t3": (3, 120, 160, 256, True, True), "spatial_time_512_60x80_t1": (1, 60, 80, 512, True, True),
              "time_512_60x80_t5": (5, 60, 80, 512, False, True)}


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("name", list(LIN_SHAPES))
def test_vae_upsample_linear2x_vs_interpolate(name, dtype):
    T, H, W, C, sp, tm = LIN_SHAPES[name]
    x = _rand(1, T, H, W, C, dtype=dtype, seed=6)
    want = EV.vae_upsample_linear2x(x, sp, tm)  # F.interpolate trilinear, as the reference calls it
    To = want.shape[1]
    buf = torch.empty(1, To + 2, *want.shape[2:], dtype=dtype, device=DEV)
    got = kernels.vae_upsample_linear2x(x, sp, tm, out=buf, t_off=2)[:, 2:]
    eq, ulp = _report(f"upsample_linear2x {name} {dtype}", got, want)
    assert torch.equal(got, kernels.vae_upsample_linear2x(x, sp, tm))
    assert eq >= 0.999 and ulp <= 1


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_vae_mix_vs_eager(dtype):
    xbuf, y = _rand(1, 11, 60, 80, 512, dtype=dtype, seed=7), _rand(1, 9, 60, 80, 512, dtype=dtype, seed=8)
    alpha = torch.sigmoid(torch.tensor([0.7], dtype=dtype, device=DEV))
    want = alpha * xbuf[:, 2:] + (1 - alpha) * y
    got = kernels.vae_mix(xbuf, y, float(alpha), float(1 - alpha), t_off=2)
    eq, _ = _report(f"mix {dtype}", got, want)
    assert eq == 1.0


# ---- the whole decoder ----
def _vae(name, dtype):
    version, cfg, _, tiling = CASES[name]
    vae = decoder_class(version)(**cfg)
    vae.load_state_dict(weights(vae.state_dict(), name))
    vae = vae.to(dtype).to(DEV).eval()
    if tiling is not None:
        apply_tiling(vae, tiling)
    return vae


def _eager(monkeypatch, vae, z):
    """The eager torch / cuDNN decoder: the same module on the kernels' stand-ins."""
    with monkeypatch.context() as m:
        for n, f in EV.stand_ins().items():
            m.setattr(kernels, n, f)
        return vae.decode(z)


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", "osp_vae.pt"))


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("name", list(CASES))
def test_osp_vae_decode_golden_within_eager16_error(monkeypatch, gold, name, dtype, no_tf32):
    vae = _vae(name, dtype)
    z = latents(name, dtype).to(DEV)
    n0 = kernels.launch_count()
    ours = vae.decode(z)
    assert kernels.launch_count() - n0 > 10
    assert list(ours.shape) == gold[f"{name}.shape"]
    eager = _eager(monkeypatch, vae, z)
    want = gold[f"{name}.fp32"].double()
    idx = sample_index(ours.numel(), name).to(DEV) if ours.numel() > want.numel() else torch.arange(ours.numel(), device=DEV)
    e_ours = float((ours.flatten()[idx].double().cpu() - want).norm())
    e_eager = float((eager.flatten()[idx].double().cpu() - want).norm())
    print(f"[decode {name} {dtype}] |ours - ref| = {e_ours:.4g}, |eager16 - ref| = {e_eager:.4g}, ratio {e_ours / e_eager:.3f}")
    assert e_ours <= 1.25 * e_eager


def test_osp_generate_with_native_vae():
    from videosys_b200.pipelines.open_sora_plan import pipeline_open_sora_plan as P

    class _ZeroDiT(torch.nn.Module):
        config = type("C", (), dict(in_channels=4, out_channels=4, caption_channels=8))()
        video_length = 3

        def reset_pab_state(self):
            pass

        def forward(self, hidden_states, **kw):
            return (torch.zeros_like(hidden_states),)

    pipe = P.OpenSoraPlanPipeline.__new__(P.OpenSoraPlanPipeline)
    pipe._config = P.OpenSoraPlanConfig(version="v110", transformer_type="65x512x512", vae=_vae("v110_res_attn3d_b2", torch.float16),
                                        transformer_config={})
    pipe._config.num_frames = 7
    pipe._device, pipe._dtype = torch.device(DEV), torch.float16
    pipe.transformer = _ZeroDiT()
    pipe.scheduler = P.PNDMScheduler()
    pipe.vae = pipe._load_vae()
    pipe._maybe_seed = lambda seed: None
    g = torch.Generator().manual_seed(0)
    out = pipe.generate(height=32, width=48, num_inference_steps=4, guidance_scale=1.0, latents=torch.randn(1, 4, 3, 4, 6, generator=g),
                        prompt_embeds=torch.randn(1, 4, 8, generator=g)).video
    assert out.dtype == torch.uint8 and tuple(out.shape) == (1, 7, 32, 48, 3)
    assert int(out.max()) > int(out.min())
