"""CogVideoX VAE decoder on the H100: each new kernel against eager torch laid out the way the reference calls it (F.pad +
F.conv3d on NCDHW, F.group_norm, F.interpolate, F.silu) in bf16 and fp16 at the released shapes, with the bit-equal
fraction and the largest error in ulps reported; repeated launches identical; the whole decoder against the reference's
fp32 outputs within 1.25x of the eager 16-bit decoder's own error."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle.gen_golden_cogvideox_vae import CASES, latents, sample_index, weights
from tests import kernels_emul_vae as EV
from videosys_b200 import kernels
from videosys_b200.models.autoencoders import AutoencoderKLCogVideoX

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]


def _ulps(got, want, *terms):
    """|got - want| in units of the 16-bit spacing at max(|got|, |want|, |terms|).  The terms are the rounded summands of
    the last eager add: where they nearly cancel, one ulp of a summand is many ulps of the result."""
    g, w = got.float(), want.float()
    mag = torch.maximum(g.abs(), w.abs())
    for t in terms:
        mag = torch.maximum(mag, t.float().abs())
    mag = mag.to(want.dtype)
    ulp = (torch.nextafter(mag, torch.full_like(mag, float("inf"))) - mag).float()
    return ((g - w).abs() / ulp).double()


def _report(what, got, want, *terms):
    u = _ulps(got, want, *terms)
    eq = float((got == want).float().mean())
    print(f"[{what}] bit-equal {100 * eq:.4f} %, max {float(u.max()):.0f} ulp")
    return eq, float(u.max())


def _rand(*shape, dtype, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (scale * torch.randn(*shape, generator=g)).to(dtype).to(DEV)


CONV_SHAPES = {  # name: (B, T, H, W, Cin, Cout, kt, residual)
    "conv_in_16to512_60x90": (1, 3, 60, 90, 16, 512, 3, False),
    "conv_512_tile30x45": (1, 3, 30, 45, 512, 512, 3, True),
    "upsample_conv2d_512_60x90": (1, 4, 60, 90, 512, 512, 1, False),
    "conv_128_240x360": (1, 2, 240, 360, 128, 128, 3, True),
    "conv_out_128to3_240x360": (1, 2, 240, 360, 128, 3, 3, False),
    "edge_64_13x21": (2, 1, 13, 21, 64, 64, 3, True),
}


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("name", list(CONV_SHAPES))
def test_vae_conv3d_vs_eager(name, dtype):
    B, T, H, W, Cin, Cout, kt, res = CONV_SHAPES[name]
    x = _rand(B, T + kt - 1, H, W, Cin, dtype=dtype, seed=1)
    w = _rand(Cout, Cin, kt, 3, 3, dtype=dtype, scale=(Cin * kt * 9) ** -0.5, seed=2)
    b = _rand(Cout, dtype=dtype, scale=0.1, seed=3)
    r = _rand(B, T, H, W, Cout, dtype=dtype, seed=4) if res else None
    wp = kernels.pack_conv_weight(w)
    xi = F.pad(x.permute(0, 4, 1, 2, 3), (1, 1, 1, 1))
    conv = F.conv3d(xi, w)
    rules = {}
    for rc in (True, False):
        want = conv + b.view(1, -1, 1, 1, 1) if rc else F.conv3d(xi, w, b)
        if res:
            want = want + r.permute(0, 4, 1, 2, 3)
        want = want.permute(0, 2, 3, 4, 1)
        got = kernels.vae_conv3d(x, wp, b, Cout, kt, resid=r, round_conv=rc)
        terms = [conv.permute(0, 2, 3, 4, 1)] + ([r] if res else [])
        rules[rc] = _report(f"{name} {dtype} round_conv={int(rc)}", got, want, *terms)
    again = kernels.vae_conv3d(x, wp, b, Cout, kt, resid=r)
    assert torch.equal(again, kernels.vae_conv3d(x, wp, b, Cout, kt, resid=r))
    # The rule the decoder uses (round_conv=True, vae_conv3d's default) matches cuDNN on >= 98 % of the elements.  The
    # rest differ where cuDNN's own fp32 sum order differs; at some 512-channel shapes its fp16 result is off by tens of
    # ulps of the largest summand, so the ulp bound is loose and the decoder-level test below bounds the effect.
    eq, ulp = rules[True]
    assert eq >= 0.98 and ulp <= 64, rules


def _eager_norm(f, gamma, beta, zyb, G):
    B, T, H, W, C = f.shape
    fi = f.permute(0, 4, 1, 2, 3)
    z = zyb.permute(0, 4, 1, 2, 3)
    zy, zb = EV._interp(z[:, :C], (T, H, W)), EV._interp(z[:, C:], (T, H, W))
    n = F.group_norm(fi, G, gamma, beta, 1e-6)
    m = n * zy
    return F.silu(m + zb).permute(0, 2, 3, 4, 1), m.permute(0, 2, 3, 4, 1), zb.permute(0, 2, 3, 4, 1)


NORM_SHAPES = {  # name: (B, T, H, W, C, Tz, h, w)
    "mid_512_60x90_t3": (1, 3, 60, 90, 512, 3, 60, 90),
    "up_256_120x180_t5": (1, 5, 120, 180, 256, 3, 60, 90),
    "up_128_240x360_t9": (1, 9, 240, 360, 128, 3, 30, 45),
    "up_128_240x360_t8": (1, 8, 240, 360, 128, 2, 30, 45),
}


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("name", list(NORM_SHAPES))
def test_vae_spatial_norm_silu_vs_eager(name, dtype):
    B, T, H, W, C, Tz, h, w = NORM_SHAPES[name]
    G = 32
    f = _rand(B, T, H, W, C, dtype=dtype, scale=2.0, seed=5) + 0.5
    gamma = _rand(C, dtype=dtype, scale=0.2, seed=6) + 1
    beta = _rand(C, dtype=dtype, scale=0.1, seed=7)
    zyb = _rand(B, Tz, h, w, 2 * C, dtype=dtype, seed=8)
    stats = kernels.vae_groupnorm_stats(f, G, 1e-6)
    assert torch.equal(stats, kernels.vae_groupnorm_stats(f, G, 1e-6))  # fixed-order reduction
    ref = EV.vae_groupnorm_stats(f, G, 1e-6)
    assert torch.allclose(stats, ref, rtol=1e-5, atol=1e-6)
    out = torch.zeros(B, T + 2, H, W, C, dtype=dtype, device=DEV)
    kernels.vae_spatial_norm_silu(f, stats, gamma, beta, zyb, out, t_off=2)
    assert torch.all(out[:, :2] == 0)
    eq, ulp = _report(f"spatial_norm_silu {name} {dtype}", out[:, 2:], *_eager_norm(f, gamma, beta, zyb, G))
    assert eq >= 0.98 and ulp <= 4


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("T,compress", [(3, True), (2, True), (1, True), (4, False)])
def test_vae_upsample2x_matches_interpolate(T, compress, dtype):
    x = _rand(1, T, 30, 45, 512, dtype=dtype, seed=9)
    got = kernels.vae_upsample2x(x, compress)
    assert torch.equal(got, EV.vae_upsample2x(x, compress))


def _vae(name, dtype):
    cfg, _, tiling = CASES[name]
    vae = AutoencoderKLCogVideoX(**cfg)
    vae.load_state_dict(weights(vae.state_dict(), name))
    vae = vae.to(dtype).to(DEV).eval()
    if tiling is not None:
        vae.enable_tiling(**tiling)
    return vae


def _eager(monkeypatch, vae, z):
    with monkeypatch.context() as m:
        for n, f in EV.stand_ins().items():
            m.setattr(kernels, n, f)
        m.setattr(kernels, "require_cuda", lambda *a, **k: None)  # the fp32 reference run
        return vae.decode(z).sample


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", "cogvideox_vae.pt"))


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("name", list(CASES))
def test_vae_decode_golden_within_eager16_error(monkeypatch, gold, name, dtype):
    vae = _vae(name, dtype)
    z = latents(name, dtype).to(DEV)
    n0 = kernels.launch_count()
    ours = vae.decode(z).sample
    assert kernels.launch_count() - n0 > 10
    eager = _eager(monkeypatch, vae, z)
    want = gold[f"{name}.fp32"].double()
    idx = sample_index(ours.numel(), name).to(DEV)
    e_ours = float((ours.flatten()[idx].double().cpu() - want).norm())
    e_eager = float((eager.flatten()[idx].double().cpu() - want).norm())
    print(f"[decode {name} {dtype}] |ours - ref| = {e_ours:.4g}, |eager16 - ref| = {e_eager:.4g}, ratio {e_ours / e_eager:.3f}")
    assert e_ours <= 1.25 * e_eager


def test_vae_decode_cogvideox_2b_shape_tiled(monkeypatch):
    """Latents [1, 16, 13, 60, 90] fp16, released widths, tiled -> [1, 3, 49, 480, 720]."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    vae = _vae("released_f3", torch.float16)
    vae.enable_tiling()
    g = torch.Generator().manual_seed(7)
    z = torch.randn(1, 16, 13, 60, 90, generator=g).to(DEV)
    ours = vae.decode(z.half()).sample
    assert tuple(ours.shape) == (1, 3, 49, 480, 720)
    eager16 = _eager(monkeypatch, vae, z.half())
    ref = _eager(monkeypatch, vae.float(), z).double()
    e_ours, e_eager = float((ours.double() - ref).norm()), float((eager16.double() - ref).norm())
    print(f"[decode 2b tiled fp16] |ours - ref32| = {e_ours:.4g}, |eager16 - ref32| = {e_eager:.4g}, ratio {e_ours / e_eager:.3f}")
    assert e_ours <= 1.25 * e_eager


def test_generate_with_native_vae_pt():
    from videosys_b200.pipelines.cogvideox import pipeline_cogvideox as P

    class _ZeroDiT(torch.nn.Module):
        config = type("C", (), dict(in_channels=16, text_embed_dim=8, use_rotary_positional_embeddings=False, patch_size=2))()

        def reset_pab_state(self):
            pass

        def forward(self, hidden_states, **kw):
            return (torch.zeros_like(hidden_states),)

    pipe = P.CogVideoXPipeline.__new__(P.CogVideoXPipeline)
    pipe._config = P.CogVideoXConfig(vae=_vae("small_f3", torch.float16), vae_tiling=False)
    pipe._device, pipe._dtype = torch.device(DEV), torch.float16
    pipe.transformer = _ZeroDiT()
    pipe.scheduler = P.CogVideoXDDIMScheduler()
    pipe.vae = pipe._load_vae()
    pipe._maybe_seed = lambda seed: None
    out = pipe.generate(height=48, width=80, num_frames=9, num_inference_steps=2, guidance_scale=1.0,
                        prompt_embeds=torch.randn(1, 4, 8), output_type="pt").video
    assert tuple(out.shape) == (1, 9, 3, 48, 80) and out.is_cuda
    assert float(out.min()) >= 0 and float(out.max()) <= 1 and torch.isfinite(out.float()).all()
