"""The VAE decoder kernels (csrc/vae_conv.cu, csrc/vae_osp.cu) element by element against float64, in bf16 and fp16.

Each arithmetic kernel is checked with the acceptance rule of tests/vae_fp64.py: the float64 core of the operation, the
reference model's eager 16-bit rounding points after it, and both neighbours legal only where the float64 value lies
within eps of a midpoint.  Every check prints its eps, the bit-equal fraction, the largest error in ulps and the largest
accepted |value - midpoint|.  Data movement (gathers, splits, merges, nearest up-sampling, the TimeUpsampleRes2x mix) is
checked bit for bit.  Inputs look like decoder activations: a DC offset, a few channels scaled x 20, post-SiLU skew."""
import pytest
import torch
import torch.nn.functional as F

from tests import kernels_emul_vae as EV
from tests import vae_fp64 as V
from videosys_b200 import kernels
from videosys_b200.models.autoencoders._common import frame_attention

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _rand(*shape, dtype, scale=1.0, offset=0.0, seed=0):
    return (offset + scale * torch.randn(*shape, generator=_gen(seed))).to(dtype).to(DEV)


def _act(*shape, dtype, seed, offset=0.3):
    """Decoder-like activations, channels last: every third channel post-SiLU, a DC offset, four channels x 20."""
    z = torch.randn(*shape, generator=_gen(seed))
    z[..., ::3] = F.silu(2 * z[..., ::3])
    z = z + offset
    z[..., :4] *= 20
    return z.to(dtype).to(DEV)


def _nan_sentinels_intact(what, buf, t0, t1):
    outside = torch.cat([buf[:, :t0], buf[:, t1:]], 1)
    assert bool(torch.isnan(outside.float()).all()), f"{what}: wrote outside frames {t0}..{t1 - 1}"


# =====================================================================================================================
# vae_conv3d
# =====================================================================================================================
CONV_CASES = {  # name: (B, T, H, W, Cin, Cout, kt, residual)
    "conv_in_16to64_13x21": (2, 1, 13, 21, 16, 64, 3, False),
    "conv_in_16to512_30x45": (1, 3, 30, 45, 16, 512, 3, False),
    "64_1x1": (2, 3, 1, 1, 64, 64, 3, True),
    "64to192_5x7": (2, 1, 5, 7, 64, 192, 3, True),
    "128_240x360": (1, 2, 240, 360, 128, 128, 3, True),
    "128to3_240x360": (1, 1, 240, 360, 128, 3, 3, False),
    "128to3_60x90_b2": (2, 3, 60, 90, 128, 3, 3, False),
    "192_13x21": (2, 3, 13, 21, 192, 192, 3, True),
    "256to128_kt1_60x90": (2, 3, 60, 90, 256, 128, 1, False),
    "512_30x45": (1, 2, 30, 45, 512, 512, 3, True),
    "512to192_kt1_5x7": (2, 1, 5, 7, 512, 192, 1, True),
    "512to64_kt1_1x1": (2, 3, 1, 1, 512, 64, 1, False),
}


def _regions(B, T, H, W):
    """Border pixels, tile-seam pixels of the 8 x 16 conv tile (not on the border) and the interior, as [B, T, H, W]."""
    y = torch.arange(H, device=DEV).view(H, 1)
    x = torch.arange(W, device=DEV).view(1, W)
    border = (y == 0) | (y == H - 1) | (x == 0) | (x == W - 1)
    seam = (((x % 16 == 0) | (x % 16 == 15)) | ((y % 8 == 0) | (y % 8 == 7))) & ~border
    interior = ~border & ~seam
    return {k: m.expand(B, T, H, W) for k, m in (("border", border), ("seam", seam), ("interior", interior))}


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", list(CONV_CASES))
def test_vae_conv3d_fp64(name, dtype):
    B, T, H, W, Cin, Cout, kt, res = CONV_CASES[name]
    x = _act(B, T + kt - 1, H, W, Cin, dtype=dtype, seed=1)
    if kt > 1:  # causal context frames unlike the T frames, so that a wrong frame offset shows
        x[:, :kt - 1] = _act(B, kt - 1, H, W, Cin, dtype=dtype, seed=11, offset=-0.8)
    w = _rand(Cout, Cin, kt, 3, 3, dtype=dtype, scale=(Cin * kt * 9) ** -0.5, seed=2)
    b = _rand(Cout, dtype=dtype, scale=0.1, seed=3)
    r = _act(B, T, H, W, Cout, dtype=dtype, seed=4) if res else None
    wp = kernels.pack_conv_weight(w)
    regions = _regions(B, T, H, W)
    failed = []
    for rc in (True, False):
        got = kernels.vae_conv3d(x, wp, b, Cout, kt, resid=r, round_conv=rc)
        ch = V.conv_chain(x, w, b, r, rc)
        for where, m in regions.items():
            if bool(m.any()) and not V.check(f"conv3d {name} {dtype} round_conv={int(rc)} {where}", got, ch, mask=m)[0]:
                failed.append((rc, where))
    assert not failed, f"outside the legal set at (round_conv, region): {failed}"


# =====================================================================================================================
# vae_groupnorm_stats against float64 mean and variance
# =====================================================================================================================
STAT_SHAPES = [(2, P, C) for C in (64, 128, 256, 512) for P in (1, 7, 4097)] + [(2, 9 * 240 * 360, 128)]
OFFSET_SIGMA = [(0, 1), (10, 1), (30, 1), (10, 0.05), (10, 0.01), (4, 0.002)]


def _check_stats(what, x, G, eps=1e-6):
    stats = kernels.vae_groupnorm_stats(x, G, eps)
    assert torch.equal(stats, kernels.vae_groupnorm_stats(x, G, eps))  # fixed-order reduction, no atomics
    B, C = x.shape[0], x.shape[-1]
    v = x.reshape(B, -1, G, C // G).transpose(1, 2).reshape(B, G, -1).double()
    mean64 = v.mean(-1)
    var64 = ((v - mean64[..., None]) ** 2).mean(-1)
    rstd64 = (var64 + eps).rsqrt()
    sd64 = var64.sqrt()
    e_mean = (stats[..., 0].double() - mean64).abs() / (mean64.abs() + sd64)
    e_rstd = (stats[..., 1].double() / rstd64 - 1).abs()
    # torch's own GroupNorm statistics on the same GPU, in the input's dtype: reported, not a bound (on a DC offset with a
    # small spread torch's fp16 rstd is itself several ulps from float64)
    xt = x.reshape(B, -1, C).transpose(1, 2).contiguous()
    _, tm, tr = torch.native_group_norm(xt, None, None, B, C, xt.shape[-1], G, eps)
    d_mean = (V.round16(stats[..., 0].double(), x.dtype) - tm.view(B, G).double()).abs() / V.ulp16(tm.view(B, G), x.dtype)
    d_rstd = (V.round16(stats[..., 1].double(), x.dtype) - tr.view(B, G).double()).abs() / V.ulp16(tr.view(B, G), x.dtype)
    print(f"[groupnorm_stats {what}] max |mean - mean64| / (|mean64| + sd64) {float(e_mean.max()):.3g}, "
          f"max rstd rel err {float(e_rstd.max()):.3g}; vs torch ({x.dtype}) mean {float(d_mean.max()):.0f} ulp, "
          f"rstd {float(d_rstd.max()):.0f} ulp")
    ok = float(e_mean.max()) <= 1e-6 and float(e_rstd.max()) <= 1e-5
    return stats, ok


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("offset,sigma", OFFSET_SIGMA)
def test_vae_groupnorm_stats_fp64(offset, sigma, dtype):
    failed = []
    for i, (B, P, C) in enumerate(STAT_SHAPES):
        x = (offset + sigma * torch.randn(B, P, C, generator=_gen(20 + i))).to(dtype).to(DEV)
        if not _check_stats(f"{dtype} offset={offset} sigma={sigma} B={B} P={P} C={C}", x, 32)[1]:
            failed.append((P, C))
    assert not failed, f"(P, C) beyond the bounds: {failed}"


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_vae_groupnorm_stats_constant_group(dtype):
    """One exactly constant group on a DC offset (and its neighbours not): rstd = eps^-1/2."""
    failed = []
    for B, P, C in STAT_SHAPES:
        x = _act(B, P, C, dtype=dtype, seed=30)
        cg = C // 32
        x[:, :, 5 * cg:6 * cg] = torch.tensor(10.0625, dtype=dtype)
        stats, ok = _check_stats(f"{dtype} constant group P={P} C={C}", x, 32)  # rstd within 1e-5 of eps^-1/2
        if not ok or not bool((stats[:, 5, 0] == 10.0625).all()):
            failed.append((P, C))
    assert not failed, f"(P, C) beyond the bounds: {failed}"


# =====================================================================================================================
# vae_spatial_norm_silu and vae_groupnorm_act, fed the kernel's own statistics
# =====================================================================================================================
NORM_CASES = {  # name: (B, T, H, W, C, Tz, h, w)
    "t5_odd_20x28_from_7x9": (2, 5, 20, 28, 128, 3, 7, 9),
    "t4_even_14x18_from_7x9": (2, 4, 14, 18, 64, 2, 7, 9),
    "t1_20x20_from_7x7": (2, 1, 20, 20, 256, 1, 7, 7),
    "t3_512_60x90": (2, 3, 60, 90, 512, 3, 60, 90),
    "t9_128_240x360": (1, 9, 240, 360, 128, 3, 30, 45),
}


def _gather(zyb, T, H, W):
    """zy, zb of zyb [B, Tz, h, w, 2C] at [B, T, H, W, C], by the reference's F.interpolate (nearest)."""
    C = zyb.shape[-1] // 2
    z = zyb.permute(0, 4, 1, 2, 3)
    return [EV._interp(z[:, i * C:(i + 1) * C], (T, H, W)).permute(0, 2, 3, 4, 1) for i in range(2)]


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", list(NORM_CASES))
def test_vae_spatial_norm_silu_fp64(name, dtype):
    B, T, H, W, C, Tz, h, w = NORM_CASES[name]
    f = _act(B, T, H, W, C, dtype=dtype, seed=5)
    gamma = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=6)
    beta = _rand(C, dtype=dtype, scale=0.1, seed=7)
    zyb = _act(B, Tz, h, w, 2 * C, dtype=dtype, seed=8, offset=0.0)
    stats = kernels.vae_groupnorm_stats(f, 32, 1e-6)
    out = torch.full((B, T + 3, H, W, C), float("nan"), dtype=dtype, device=DEV)
    kernels.vae_spatial_norm_silu(f, stats, gamma, beta, zyb, out, t_off=2)
    _nan_sentinels_intact("spatial_norm_silu", out, 2, 2 + T)
    zy, zb = _gather(zyb, T, H, W)
    ch = V.spatial_norm_silu_chain(V.gn_affine_chain(f, stats, gamma, beta), zy, zb)
    V.assert_legal(f"spatial_norm_silu {name} {dtype}", out[:, 2:2 + T], ch)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", [n for n in NORM_CASES if n != "t9_128_240x360"])
def test_vae_spatial_norm_nearest_gather_exact(name, dtype):
    """gamma = 0, beta = 1 make the norm exactly 1 and zb = 0, so the output is silu of the gathered zy, which encodes
    the source (frame, row, column) + 1 in three channel phases: a wrong source index is many ulps off."""
    B, T, H, W, C, Tz, h, w = NORM_CASES[name]
    f = _act(B, T, H, W, C, dtype=dtype, seed=5)
    zt = torch.arange(Tz).view(1, Tz, 1, 1).expand(B, Tz, h, w)
    zy_ = torch.arange(h).view(1, 1, h, 1).expand(B, Tz, h, w)
    zx = torch.arange(w).view(1, 1, 1, w).expand(B, Tz, h, w)
    code = torch.stack([zt, zy_, zx], -1).repeat(1, 1, 1, 1, -(-C // 3))[..., :C] + 1.0
    zyb = torch.cat([code, torch.zeros_like(code)], -1).to(dtype).to(DEV)
    gamma, beta = torch.zeros(C, dtype=dtype, device=DEV), torch.ones(C, dtype=dtype, device=DEV)
    stats = kernels.vae_groupnorm_stats(f, 32, 1e-6)
    out = torch.full((B, T + 2, H, W, C), float("nan"), dtype=dtype, device=DEV)
    kernels.vae_spatial_norm_silu(f, stats, gamma, beta, zyb, out, t_off=1)
    _nan_sentinels_intact("spatial_norm_silu gather", out, 1, 1 + T)
    zy, zb = _gather(zyb, T, H, W)
    ch = V.spatial_norm_silu_chain(V.gn_affine_chain(f, stats, gamma, beta), zy, zb)
    V.assert_legal(f"spatial_norm gather {name} {dtype}", out[:, 1:1 + T], ch)


GN_CASES = {"512_60x80_t3": (2, 3, 60, 80, 512), "128_240x320_t2": (1, 2, 240, 320, 128), "64_5x7_t1": (2, 1, 5, 7, 64)}


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("act", [True, False], ids=["act", "noact"])
@pytest.mark.parametrize("name", list(GN_CASES))
def test_vae_groupnorm_act_fp64(name, act, dtype):
    B, T, H, W, C = GN_CASES[name]
    x = _act(B, T, H, W, C, dtype=dtype, seed=1)
    gamma, beta = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=2), _rand(C, dtype=dtype, scale=0.1, seed=3)
    stats = kernels.vae_groupnorm_stats(x, 32, 1e-6)
    buf = torch.full((B, T + 3, H, W, C), float("nan"), dtype=dtype, device=DEV)
    kernels.vae_groupnorm_act(x, stats, gamma, beta, out=buf, t_off=2, act=act)
    _nan_sentinels_intact("groupnorm_act", buf, 2, 2 + T)
    ch = V.gn_affine_chain(x, stats, gamma, beta)
    if act:
        ch = V.sigmoid_act_chain(ch)
    V.assert_legal(f"groupnorm_act {name} act={int(act)} {dtype}", buf[:, 2:2 + T], ch)


# =====================================================================================================================
# Open-Sora-Plan attention: split / merge bit for bit, the softmax and the whole path against float64
# =====================================================================================================================
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("T", [1, 2, 3])
@pytest.mark.parametrize("C", [256, 512])
@pytest.mark.parametrize("mixed", [False, True], ids=["fix", "mixed"])
def test_vae_attn_split_merge_bit_exact(mixed, C, T, dtype):
    B = 2
    for H, W in ((3, 5), (10, 10), (60, 80)):
        qkv = _act(B, T, H, W, 3 * C, dtype=dtype, seed=40 + H)
        q, k, vt = kernels.vae_attn_split(qkv, C, mixed)
        rq, rk, rvt = EV.vae_attn_split(qkv, C, mixed)  # torch reshape / permute, zero padded
        what = f"attn_split mixed={int(mixed)} C={C} T={T} P={H * W} {dtype}"
        V.assert_bit_exact(what + " q", q, rq)
        V.assert_bit_exact(what + " k", k, rk)
        V.assert_bit_exact(what + " vt", vt, rvt)
        o = _act(B * T, H * W, C, dtype=dtype, seed=50 + H)
        want = o.permute(0, 2, 1).reshape(B, C, T, H, W).permute(0, 2, 3, 4, 1)  # AttnBlock3D's h_.reshape(b, c, t, h, w)
        V.assert_bit_exact(f"attn_merge C={C} T={T} P={H * W} {dtype}", kernels.vae_attn_merge(o, B, T, H, W), want.contiguous())


def _score_rows(P, Pp, dtype, scale):
    """Rows of raw scores S [rows, Pp]: random, peaked (+40 after scaling), constant, very negative, near the fp16 top."""
    g = _gen(60 + P)
    rand = 8 * torch.randn(4, Pp, generator=g)
    peaked = torch.randn(4, Pp, generator=g)
    peaked[torch.arange(4), torch.randint(0, P, (4,), generator=g)] += 40 / scale
    const = torch.full((2, Pp), 3.0)
    neg = -30000 + 50 * torch.randn(2, Pp, generator=g)
    top = 65504 - 32 * torch.randint(0, 200, (2, Pp), generator=g).float()
    S = torch.cat([rand, peaked, const, neg, top]).to(dtype)
    S[:, P:] = torch.randn(S.shape[0], Pp - P, generator=g).to(dtype)  # garbage in the padding columns
    return S.to(DEV)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("P", [1, 15, 257, 4800])
def test_vae_attn_softmax_fp64(P, dtype):
    Pp = -(-P // 8) * 8
    scale = 512 ** -0.5
    S = _score_rows(P, Pp, dtype, scale)
    got = kernels.vae_attn_softmax_(S.clone(), P, scale)
    s16 = (S[:, :P].float() * scale).to(dtype).double()  # the reference's eager w_ * c ** -0.5, one rounding
    p = torch.softmax(s16, -1)
    d = (s16 - s16.max(-1, keepdim=True).values).abs()
    # fp32 exp (2 ulps) of an fp32 difference, a fixed-order sum of positive terms, one division; subnormal exp results
    eps = p * V.U32 * (P / 256 + 24 + 2 * d) + 2.0**-148
    V.assert_legal(f"attn_softmax P={P} {dtype}", got[:, :P], V.Chain.start(p, eps, dtype))
    V.assert_bit_exact(f"attn_softmax padding P={P} {dtype}", got[:, P:], torch.zeros_like(got[:, P:]))
    assert torch.equal(got, kernels.vae_attn_softmax_(S.clone(), P, scale))


ATTN_CASES = {"fix_60x80_t1_c512": (1, 60, 80, 512, False), "mixed_20x30_t2_c512": (2, 20, 30, 512, True),
              "mixed_15x16_t3_c256": (3, 15, 16, 256, True), "fix_3x5_t2_c256": (2, 3, 5, 256, False)}


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", list(ATTN_CASES))
def test_vae_attention_path_fp64(name, dtype, monkeypatch):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    T, H, W, C, mixed = ATTN_CASES[name]
    qkv = _rand(2, T, H, W, 3 * C, dtype=dtype, scale=1.5, seed=70)
    ours = frame_attention(qkv, C, mixed)
    eager = EV.eager_attention(qkv, C, mixed)
    exact = EV.eager_attention(qkv.double(), C, mixed)
    err, err_eager = (ours.double() - exact).abs(), (eager.double() - exact).abs()
    print(f"[attention {name} {dtype}] max|err| vs fp64 {float(err.max()):.3e} (eager16 {float(err_eager.max()):.3e}), "
          f"mean {float(err.mean()):.3e} (eager16 {float(err_eager.mean()):.3e})")
    bf = dtype == torch.bfloat16
    # the bound of the flash-attention test, widened by twice the error of the reference's own 16-bit chain at the same
    # element: that chain rounds the scores and the probabilities to 16 bits, which flash attention does not
    tol = (2.0**-7 if bf else 2.0**-9) * exact.abs().clamp_min(0.02) + (2e-3 if bf else 1e-3) + 2 * err_eager
    bad = err > tol
    assert not bool(bad.any()), f"{int(bad.sum())} elements beyond the bound, first at {bad.nonzero()[0].tolist()}"
    assert float(err.mean()) <= 2.0 * float(err_eager.mean()) + 1e-5


# =====================================================================================================================
# vae_upsample_linear2x against a float64 trilinear of the 16-bit input; vae_upsample2x and vae_mix bit for bit
# =====================================================================================================================
LIN_CASES = {  # name: (B, T, H, W, C, spatial, temporal)
    "1x1_t2_both": (2, 2, 1, 1, 64, True, True),
    "1x1_t1_spatial": (2, 1, 1, 1, 64, True, False),
    "5x7_t1_both": (2, 1, 5, 7, 256, True, True),
    "13x21_t3_spatial": (2, 3, 13, 21, 128, True, False),
    "12x20_t4_temporal": (2, 4, 12, 20, 512, False, True),
    "60x80_t3_both": (1, 3, 60, 80, 256, True, True),
}


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", list(LIN_CASES))
def test_vae_upsample_linear2x_fp64(name, dtype):
    B, T, H, W, C, sp, tm = LIN_CASES[name]
    x = _act(B, T, H, W, C, dtype=dtype, seed=80)
    v = EV.vae_upsample_linear2x(x.double(), sp, tm)  # F.interpolate trilinear in float64, frames 1.. on their own
    mag = EV.vae_upsample_linear2x(x.double().abs(), sp, tm)  # sum of |weight * tap|
    To = v.shape[1]
    buf = torch.full((B, To + 3, *v.shape[2:]), float("nan"), dtype=dtype, device=DEV)
    kernels.vae_upsample_linear2x(x, sp, tm, out=buf, t_off=2)
    _nan_sentinels_intact("upsample_linear2x", buf, 2, 2 + To)
    V.assert_legal(f"upsample_linear2x {name} {dtype}", buf[:, 2:2 + To], V.Chain.start(v, 4 * V.U32 * mag, dtype))


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("compress", [True, False], ids=["compress_time", "spatial"])
@pytest.mark.parametrize("T", [1, 2, 3, 4, 5])
def test_vae_upsample2x_bit_exact(T, compress, dtype):
    for H, W, C in ((5, 7, 64), (30, 45, 128)):
        x = _act(2, T, H, W, C, dtype=dtype, seed=90 + T)
        V.assert_bit_exact(f"upsample2x T={T} compress={int(compress)} {H}x{W} {dtype}", kernels.vae_upsample2x(x, compress),
                           EV.vae_upsample2x(x, compress))


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("T", [1, 2, 3, 4, 5])
def test_vae_mix_bit_exact(T, dtype):
    xbuf, y = _act(2, T + 3, 12, 20, 128, dtype=dtype, seed=100), _act(2, T, 12, 20, 128, dtype=dtype, seed=101)
    alpha = torch.sigmoid(torch.tensor([0.7], dtype=dtype, device=DEV))
    a, oma = float(alpha), float(1 - alpha)
    V.assert_bit_exact(f"mix T={T} {dtype}", kernels.vae_mix(xbuf, y, a, oma, t_off=2), EV.vae_mix(xbuf, y, a, oma, t_off=2))
