"""The float64 acceptance rule of tests/vae_fp64.py on small CPU tensors: it accepts the reference chains evaluated by
torch's eager fp32 / 16-bit ops, and it rejects the kernel bugs it is there to catch (one element off by an ulp, the
wrong rounding mode, a tap missing on the image border, the wrong causal context frame, one group's rstd off by an ulp).
Neither blind nor over-strict, without a GPU."""
import pytest
import torch
import torch.nn.functional as F

from tests import kernels_emul_vae as EV
from tests import vae_fp64 as V

DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]


def _rand(*shape, dtype, scale=1.0, offset=0.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (offset + scale * torch.randn(*shape, generator=g)).to(dtype)


def _conv_case(dtype, kt=3, T=2):
    B, H, W, Cin, Cout = 2, 5, 7, 16, 8
    x = _rand(B, T + kt - 1, H, W, Cin, dtype=dtype, offset=0.3, seed=1)
    x[..., :2] *= 20  # a few large channels, as in decoder activations
    w = _rand(Cout, Cin, kt, 3, 3, dtype=dtype, scale=(Cin * kt * 9) ** -0.5, seed=2)
    b = _rand(Cout, dtype=dtype, scale=0.1, seed=3)
    r = _rand(B, T, H, W, Cout, dtype=dtype, seed=4)
    return x, w, b, r


def _eager_conv(x, w, b, r, round_conv):
    """The reference's eager chain on the CPU: fp32 convolution, 16-bit bias add (or fp32 with the bias), 16-bit add."""
    dt = x.dtype
    xi = F.pad(x.permute(0, 4, 1, 2, 3).float(), (1, 1, 1, 1))
    if round_conv:
        y = F.conv3d(xi, w.float()).to(dt) + b.view(1, -1, 1, 1, 1)
    else:
        y = F.conv3d(xi, w.float(), b.float()).to(dt)
    return (y + r.permute(0, 4, 1, 2, 3)).permute(0, 2, 3, 4, 1)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_round16_matches_torch_casts(dtype):
    g = torch.Generator().manual_seed(0)
    v = torch.cat([torch.randn(20000, generator=g, dtype=torch.float64) * 10 ** torch.randint(-6, 5, (20000,), generator=g),
                   torch.tensor([0.0, -0.0, 1e-9, 65504.0, 65519.0, 65520.0, 3e38])])
    # fp32 values: one cast to 16 bits is correctly rounded, so it must agree with the exact float64 rounding
    f = v.float()
    assert torch.equal(V.round16(f.double(), dtype), f.to(dtype).double())
    u = V.ulp16(torch.tensor([1.0, 1.5, 2.0, 0.0]), dtype)
    p = V.fmt(dtype)[0]
    assert u.tolist()[:3] == [2.0 ** (1 - p), 2.0 ** (1 - p), 2.0 ** (2 - p)]


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_tie_within_eps_accepts_both_neighbours(dtype):
    p = V.fmt(dtype)[0]
    mid = torch.tensor([1.0 + 2.0**-p], dtype=torch.float64)  # halfway between 1 and its upper neighbour
    up = 1.0 + 2.0 ** (1 - p)
    for v, eps, legal in [(mid, 0.0, [1.0]), (mid + 2.0**-30, 2.0**-29, [1.0, up]), (mid + 2.0**-28, 2.0**-29, [up])]:
        ch = V.Chain.start(v, eps, dtype)
        for g in (1.0, up):
            ok, _ = V.check("tie", torch.tensor([g], dtype=dtype), ch, verbose=False)
            assert ok == (g in legal), (float(v), eps, g)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("round_conv", [True, False])
def test_conv_chain_accepts_eager_fp32(dtype, round_conv):
    x, w, b, r = _conv_case(dtype)
    ch = V.conv_chain(x, w, b, r, round_conv)
    V.assert_legal(f"eager conv rc={int(round_conv)}", _eager_conv(x, w, b, r, round_conv), ch)
    ch = V.conv_chain(x, w, b, None, round_conv)
    xi = F.pad(x.permute(0, 4, 1, 2, 3).float(), (1, 1, 1, 1))
    y = F.conv3d(xi, w.float()).to(dtype) + b.view(1, -1, 1, 1, 1) if round_conv else F.conv3d(xi, w.float(), b.float()).to(dtype)
    V.assert_legal("eager conv no residual", y.permute(0, 2, 3, 4, 1), ch)


def _rejects(what, got, chain):
    ok, st = V.check(what, got, chain)
    assert not ok, f"{what} was accepted"
    return st


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_rejects_one_ulp_on_a_non_tie(dtype):
    x, w, b, r = _conv_case(dtype)
    ch = V.conv_chain(x, w, b, r)
    got = _eager_conv(x, w, b, r, True).double()
    # the element whose float64 value is farthest from a midpoint, i.e. closest to its 16-bit value
    dist = (ch.v - ch.near).abs() / V.ulp16(ch.near, dtype)
    i = int(torch.argmin(dist.flatten()))
    flat = got.flatten().clone()
    flat[i] += torch.sign(flat[i]) * V.ulp16(flat[i], dtype)  # the neighbour away from zero
    st = _rejects("one ulp", flat.view_as(got).to(dtype), ch)
    assert st["bad"] == 1


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_rejects_round_toward_zero(dtype):
    x, w, b, r = _conv_case(dtype)
    ch = V.conv_chain(x, w, b, r)
    xi = F.pad(x.permute(0, 4, 1, 2, 3).float(), (1, 1, 1, 1))
    y = (F.conv3d(xi, w.float()).to(dtype) + b.view(1, -1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    last = y.float() + r.float()  # the last add in fp32, then truncated instead of rounded
    _rejects("round toward zero", V.round16(last.double(), dtype, mode="zero").to(dtype), ch)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_rejects_missing_tap_on_last_column(dtype):
    x, w, b, r = _conv_case(dtype)
    ch = V.conv_chain(x, w, b, r)
    got = _eager_conv(x, w, b, r, True)
    wm = w.clone()
    wm[:, :, 2, 1, 0] = 0  # the current frame's tap at (y, x - 1)
    bad = _eager_conv(x, wm, b, r, True)
    got[:, :, :, -1] = bad[:, :, :, -1]
    st = _rejects("missing tap, last column", got, ch)
    interior = torch.ones(got.shape[:4], dtype=torch.bool)
    interior[:, :, :, -1] = False
    assert V.check("missing tap, other columns", got, ch, mask=interior)[0]
    assert st["bad"] > 0


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_rejects_wrong_context_frame(dtype):
    x, w, b, r = _conv_case(dtype, kt=3, T=1)
    ch = V.conv_chain(x, w, b, r)
    xm = x.clone()
    xm[:, 0] = x[:, 1]  # dz = 0 reads the second context frame
    _rejects("wrong context frame", _eager_conv(xm, w, b, r, True), ch)


def _norm_case(dtype):
    B, T, H, W, C, G = 2, 3, 6, 10, 64, 32
    f = _rand(B, T, H, W, C, dtype=dtype, scale=2.0, offset=0.5, seed=5)
    gamma = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=6)
    beta = _rand(C, dtype=dtype, scale=0.1, seed=7)
    zyb = _rand(B, 2, 3, 5, 2 * C, dtype=dtype, seed=8)
    stats = EV.vae_groupnorm_stats(f, G, 1e-6)
    return f, gamma, beta, zyb, stats


def _norm_chain(f, gamma, beta, zyb, stats):
    B, T, H, W, C = f.shape
    z = zyb.permute(0, 4, 1, 2, 3)
    zy, zb = (EV._interp(z[:, i * C:(i + 1) * C], (T, H, W)).permute(0, 2, 3, 4, 1) for i in range(2))
    return V.spatial_norm_silu_chain(V.gn_affine_chain(f, stats, gamma, beta), zy, zb)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_norm_chains_accept_eager(dtype):
    f, gamma, beta, zyb, stats = _norm_case(dtype)
    out = torch.empty_like(f)
    V.assert_legal("eager spatial norm silu", EV.vae_spatial_norm_silu(f, stats, gamma, beta, zyb, out), _norm_chain(f, gamma, beta, zyb, stats))
    n = V.gn_affine_chain(f, stats, gamma, beta)
    full = F.group_norm(f.permute(0, 4, 1, 2, 3).float(), 32, gamma.float(), beta.float(), 1e-6)  # the affine form is GroupNorm
    assert float((full.permute(0, 2, 3, 4, 1).double() - n.v).abs().max()) < 0.05
    mean = stats[..., 0].to(dtype).float().repeat_interleave(2, 1).view(2, 1, 1, 1, 64)
    rstd = stats[..., 1].to(dtype).float().repeat_interleave(2, 1).view(2, 1, 1, 1, 64)
    a = rstd * gamma.float()
    n16 = (a * f.float() + (beta.float() - a * mean)).to(dtype)
    V.assert_legal("eager groupnorm", n16, n)
    V.assert_legal("eager groupnorm + x * sigmoid(x)", n16 * torch.sigmoid(n16), V.sigmoid_act_chain(n))


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_rejects_one_group_rstd_off_by_one_ulp(dtype):
    f, gamma, beta, zyb, stats = _norm_case(dtype)
    ch = _norm_chain(f, gamma, beta, zyb, stats)
    bad = stats.clone()
    r16 = V.round16(stats[1, 5, 1].double(), dtype)
    bad[1, 5, 1] = float(r16 + V.ulp16(r16, dtype))
    got = EV.vae_spatial_norm_silu(f, bad, gamma, beta, zyb, torch.empty_like(f))
    st = _rejects("rstd of one group + 1 ulp", got, ch)
    in_group = torch.zeros(f.shape, dtype=torch.bool)
    in_group[1, ..., 10:12] = True
    assert V.check("other groups", got, ch, mask=~in_group)[0]
    assert st["bad"] > 0
