"""The float64 reference chains of tests/dit_fp64.py on small CPU tensors, in bf16 and fp16: every chain accepts the eager
fp32 / 16-bit evaluation of its operation (the stand-ins of tests/kernels_emul*.py, or a few lines of torch written to the
kernel's rounding points), and rejects a seeded mutation of it, one per class of kernel bug.  This is the evidence that
tests/test_dit_kernels_fp64_gpu.py is neither blind nor over-strict, without a GPU."""
import pytest
import torch
import torch.nn.functional as F

from tests import dit_fp64 as R
from tests import kernels_emul as E
from tests import kernels_emul_ds as EDS
from tests import kernels_emul_kvc as EKV
from tests import vae_fp64 as V

DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]
both = pytest.mark.parametrize("dtype", DTYPES, ids=IDS)


def _rand(*shape, dtype, scale=1.0, offset=0.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (offset + scale * torch.randn(*shape, generator=g)).to(dtype)


def _hidden(*shape, dtype, seed, offset=0.3, scale=1.0):
    """DiT-like hidden states: a DC offset and four channels x 20."""
    z = offset + torch.randn(*shape, generator=torch.Generator().manual_seed(seed))
    z[..., 3:7] *= 20
    return (scale * z).to(dtype)


def _rejects(what, got, chain, mask=None):
    ok, st = V.check(what, got, chain, mask)
    assert not ok and st["bad"] > 0, f"{what} was accepted"
    return st


def _differs(what, got, want):
    assert got.dtype == want.dtype and not torch.equal(got.view(torch.int16), want.view(torch.int16)), f"{what} was accepted"
    with pytest.raises(AssertionError):
        V.assert_bit_exact(what, got, want)


# ---------------------------------------------------------------------------------------------------------------------
# ln_modulate / ln_modulate_affine
# ---------------------------------------------------------------------------------------------------------------------
B, T, S, C = 2, 3, 5, 64


def _ln_case(dtype, scale=1.0):
    x = _hidden(B, T, S, C, dtype=dtype, seed=1, scale=scale)
    mod = _rand(2, B, 6, C, dtype=dtype, scale=0.5, seed=2)
    mask = torch.tensor([[1, 0, 1], [0, 1, 1]], dtype=torch.uint8)
    gamma = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=3)
    beta = _rand(C, dtype=dtype, scale=0.1, seed=4)
    return x, mod, mask, gamma, beta


def _ln_eager(x, mod, mask, shift_row, scale_row, eps, gamma=None, beta=None, drop_eps=False, bessel=False, short_mean=False,
              unrounded_g=False, truncate=False):
    """The kernel's rounding points in fp32 torch ops, with the bugs to inject."""
    dt = x.dtype
    xf = x.float()
    mean = xf[..., :C - 8 if short_mean else C].mean(-1, keepdim=True)
    var = ((xf - mean) ** 2).sum(-1, keepdim=True) / (C - 1 if bessel else C)
    n = (xf - mean) * torch.rsqrt(var + (0.0 if drop_eps else eps))
    if gamma is not None:
        n = n * gamma.float() + beta.float()
    n = n.to(dt)
    scale = E._mod_row(mod, mask, scale_row, B, T, C, dt)
    shift = E._mod_row(mod, mask, shift_row, B, T, C, dt)
    m = (n.float() * (1 + scale.float())).to(dt) if unrounded_g else n * (1 + scale)
    if truncate:
        return V.round16(m.double() + shift.double(), dt, mode="zero").to(dt)
    return m + shift


@both
@pytest.mark.parametrize("affine", [False, True], ids=["plain", "affine"])
@pytest.mark.parametrize("rows", [(0, 1), (3, 4), (1, 0)])
def test_ln_modulate_chain_accepts_eager(rows, affine, dtype):
    x, mod, mask, gamma, beta = _ln_case(dtype)
    gb = dict(gamma=gamma, beta=beta) if affine else {}
    for m in (None, mask):
        for eps in (1e-6, 1e-5):
            ch = R.ln_modulate_chain(x, mod, m, *rows, B, T, S, eps=eps, **gb)
            V.assert_legal("stand-in", E.ln_modulate(x, mod, m, *rows, B, T, S, eps=eps, **gb), ch)
            V.assert_legal("fp32 torch ops", _ln_eager(x, mod, m, *rows, eps, **gb), ch)


@both
@pytest.mark.parametrize("offset,sigma", [(10, 1), (30, 1), (10, 0.05), (4, 0.002), (0, 0)])
def test_ln_modulate_chain_accepts_eager_on_hard_statistics(offset, sigma, dtype):
    """A large DC offset with a small spread, down to the constant row (rstd = eps^-1/2)."""
    x = _rand(B, T, S, C, dtype=dtype, scale=sigma, offset=offset, seed=5)
    _, mod, mask, gamma, beta = _ln_case(dtype)
    V.assert_legal("plain", _ln_eager(x, mod, mask, 0, 1, 1e-6), R.ln_modulate_chain(x, mod, mask, 0, 1, B, T, S))
    V.assert_legal("affine", _ln_eager(x, mod, mask, 0, 1, 1e-6, gamma, beta),
                   R.ln_modulate_chain(x, mod, mask, 0, 1, B, T, S, gamma=gamma, beta=beta))


@both
def test_rejects_one_ulp_on_a_non_tie(dtype):
    x, mod, mask, _, _ = _ln_case(dtype)
    ch = R.ln_modulate_chain(x, mod, mask, 0, 1, B, T, S)
    got = _ln_eager(x, mod, mask, 0, 1, 1e-6).double().flatten()
    single = (ch.lo == ch.hi).flatten()  # one legal value
    i = int(single.nonzero()[7])
    got[i] += V.ulp16(got[i], dtype)
    assert _rejects("one ulp", got.view(B, T, S, C).to(dtype), ch)["bad"] == 1


@both
@pytest.mark.parametrize("bug", ["truncate", "drop_eps", "bessel", "short_mean", "unrounded_g"])
def test_rejects_ln_modulate_arithmetic_bug(bug, dtype):
    # small activations, so that eps = 1e-5 is a visible part of var + eps
    x, mod, mask, gamma, beta = _ln_case(dtype, scale=0.01 if bug == "drop_eps" else 1.0)
    for gb in ({}, dict(gamma=gamma, beta=beta)):
        ch = R.ln_modulate_chain(x, mod, mask, 0, 1, B, T, S, eps=1e-5, **gb)
        V.assert_legal(f"without {bug}", _ln_eager(x, mod, mask, 0, 1, 1e-5, **gb), ch)
        _rejects(bug, _ln_eager(x, mod, mask, 0, 1, 1e-5, **gb, **{bug: True}), ch)


@both
def test_rejects_select_shifted_by_one_frame_and_wrong_row(dtype):
    x, mod, mask, _, _ = _ln_case(dtype)
    ch = R.ln_modulate_chain(x, mod, mask, 0, 1, B, T, S)
    st = _rejects("select one frame late", _ln_eager(x, mod, mask.flatten().roll(1).view(B, T), 0, 1, 1e-6), ch)
    moved = (mask != mask.flatten().roll(1).view(B, T)).view(B, T, 1, 1).expand(B, T, S, C)
    assert st["bad"] > 0 and V.check("other frames", _ln_eager(x, mod, mask.flatten().roll(1).view(B, T), 0, 1, 1e-6), ch, mask=~moved)[0]
    _rejects("t / t0 swapped", _ln_eager(x, mod, 1 - mask, 0, 1, 1e-6), ch)
    _rejects("scale row + 1", _ln_eager(x, mod, mask, 0, 2, 1e-6), ch)
    _rejects("shift row + 1", _ln_eager(x, mod, mask, 1, 1, 1e-6), ch)
    _rejects("the other sample's rows", _ln_eager(x, mod.flip(1), mask, 0, 1, 1e-6), ch)


# ---------------------------------------------------------------------------------------------------------------------
# modulation_table, gate_residual, residual_add, gate_residual_unshuffle: one legal value each
# ---------------------------------------------------------------------------------------------------------------------
@both
def test_exact_refs_equal_eager_and_differ_from_mutations(dtype):
    x, mod, mask, _, _ = _ln_case(dtype)
    y = _hidden(B, T, S, C, dtype=dtype, seed=6)
    for rows in (6, 2):
        table = _rand(rows, C, dtype=dtype, seed=7)
        t, t0 = _rand(B, rows * C, dtype=dtype, seed=8), _rand(B, rows * C, dtype=dtype, seed=9)
        V.assert_bit_exact("table", R.modulation_table_ref(table, t, t0), E.modulation_table(table, t, t0))
        V.assert_bit_exact("table, no t0", R.modulation_table_ref(table, t, None), E.modulation_table(table, t, None))
        _differs("t0 ignored", E.modulation_table(table, t, None), R.modulation_table_ref(table, t, t0))
        _differs("row stride", E.modulation_table(table.flip(0), t, t0), R.modulation_table_ref(table, t, t0))
    for m in (None, mask):
        cache, out = R.gate_residual_ref(x, y, mod, m, 2, B, T, S)
        c2 = torch.empty_like(x)
        V.assert_bit_exact("gate_residual", E.gate_residual(x, y, mod, m, 2, B, T, S, cache_out=c2), out)
        V.assert_bit_exact("cache", c2, cache)
    fused = (x.float() + E._mod_row(mod, mask, 2, B, T, C, dtype).float() * y.float()).to(dtype)  # gate * y not rounded
    _differs("gated value not rounded", fused, out)
    _differs("gate row 5", E.gate_residual(x, y, mod, mask, 5, B, T, S), out)
    _differs("mask ignored", E.gate_residual(x, y, mod, None, 2, B, T, S), out)
    V.assert_bit_exact("residual_add", E.residual_add(x, y), R.residual_add_ref(x, y))
    _differs("truncated add", V.round16(x.double() + y.double(), dtype, mode="zero").to(dtype), R.residual_add_ref(x, y))


@both
@pytest.mark.parametrize("down", [(2, 2, 2), (1, 2, 2), (2, 1, 3)])
def test_unshuffle_ref_equals_eager_and_rejects_swapped_axes(down, dtype):
    Bq, Tq, Hq, Wq = 2, 4, 4, 6
    N = Tq * Hq * Wq
    x = _hidden(Bq, N, C, dtype=dtype, seed=1)
    mod = _rand(2, Bq, 6, C, dtype=dtype, scale=0.5, seed=2)
    y = _rand(Bq * down[0] * down[1] * down[2], N // (down[0] * down[1] * down[2]), C, dtype=dtype, seed=3)
    want = R.gate_residual_unshuffle_ref(x, y, mod, 2, Bq, Tq, Hq, Wq, down)
    V.assert_bit_exact("unshuffle", EDS.gate_residual_unshuffle(x, y, mod, 2, Bq, Tq, Hq, Wq, down), want)
    # shuffle_rows is the inverse map
    nat = _rand(Bq, Tq, Hq, Wq, C, dtype=dtype, seed=4)
    idx = R.unshuffle_index(Bq, Tq, Hq, Wq, down)
    V.assert_bit_exact("inverse", R.shuffle_rows(nat, Bq, Tq, Hq, Wq, down).reshape(-1, C)[idx], nat.reshape(-1, C))
    _differs("h and w sub-grids swapped", EDS.gate_residual_unshuffle(x, y, mod, 2, Bq, Tq, Wq, Hq, (down[0], down[2], down[1])), want)


# ---------------------------------------------------------------------------------------------------------------------
# q / k normalisation and RoPE
# ---------------------------------------------------------------------------------------------------------------------
def _qk_case(dtype, D, H=3, Sq=4, Tq=3, rows=None):
    rows = Sq * Tq * 2 - 5 if rows is None else rows  # not a multiple of S * T
    qkv = _rand(rows, 3, H, D, dtype=dtype, offset=0.4, seed=10)
    qkv[:, :, 0] += 2  # a head with a DC offset
    qkv[:, :, -1, 5] *= 50  # a head with one massive channel
    wq = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=11)
    wk = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=12)
    ang = torch.arange(Tq).view(Tq, 1) * (10000.0 ** (-torch.arange(0, D, 2) / D)).repeat_interleave(2).view(1, D)
    return qkv, wq, wk, ang.cos().contiguous(), ang.sin().contiguous(), Sq, Tq


@both
@pytest.mark.parametrize("D", [64, 72])
def test_qk_rmsnorm_chain_accepts_eager(D, dtype):
    qkv, wq, wk, cos, sin, Sq, Tq = _qk_case(dtype, D)
    for w in ((wq, wk), (None, None)):
        for rope in ((None, None), (cos, sin)):
            if w[0] is None and rope[0] is None:
                continue
            kw = dict(rope_cos=rope[0], rope_sin=rope[1], pos_div=Sq, pos_mod=Tq)
            got = E.qk_rmsnorm_(qkv.clone(), *w, 3, D, **kw)
            R.assert_qk(f"D={D} norm={w[0] is not None} rope={rope[0] is not None}", got, qkv, R.qk_rmsnorm_chain(qkv, *w, 3, D, **kw))
    got = E.qk_rmsnorm_(qkv.clone(), wq, wk, 3, D, rope_cos=cos[:1], rope_sin=sin[:1], pos_div=1, pos_mod=1)  # T = 1
    R.assert_qk("T=1", got, qkv, R.qk_rmsnorm_chain(qkv, wq, wk, 3, D, rope_cos=cos[:1], rope_sin=sin[:1]))


@both
def test_rejects_qk_rmsnorm_bugs(dtype):
    D = 72
    qkv, wq, wk, cos, sin, Sq, Tq = _qk_case(dtype, D)
    qkv = (qkv.float() * 0.002).to(dtype)  # small heads: eps is a visible part of mean(x^2) + eps
    ch = R.qk_rmsnorm_chain(qkv, wq, wk, 3, D, eps=1e-5)
    R.assert_qk("as is", E.qk_rmsnorm_(qkv.clone(), wq, wk, 3, D, eps=1e-5), qkv, ch)
    _rejects("eps left out", E.qk_rmsnorm_(qkv.clone(), wq, wk, 3, D, eps=0.0).view(-1, 3, 3, D)[:, :2], ch)
    _rejects("wq and wk swapped", E.qk_rmsnorm_(qkv.clone(), wk, wq, 3, D, eps=1e-5).view(-1, 3, 3, D)[:, :2], ch)
    xf = qkv.float()[:, :2]
    ms = xf[..., :D - 8].pow(2).sum(-1, keepdim=True) / D  # the last 8-channel vector left out of the sum
    short = torch.stack([wq, wk]).view(1, 2, 1, D) * (xf * torch.rsqrt(ms + 1e-5)).to(dtype)
    _rejects("last vector dropped", short, ch)
    fused = (torch.stack([wq, wk]).view(1, 2, 1, D).float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5))).to(dtype)
    _rejects("h not rounded before the weight", fused, ch)
    touched = E.qk_rmsnorm_(qkv.clone(), wq, wk, 3, D, eps=1e-5)
    touched.view(-1, 3, 3, D)[4, 2, 1, 3] *= 2
    with pytest.raises(AssertionError):
        R.assert_qk("v modified", touched, qkv, ch)


@both
@pytest.mark.parametrize("norm", [True, False], ids=["norm+rope", "rope_only"])
def test_rejects_rope_bugs(norm, dtype):
    D = 64
    qkv, wq, wk, cos, sin, Sq, Tq = _qk_case(dtype, D)
    w = (wq, wk) if norm else (None, None)
    ch = R.qk_rmsnorm_chain(qkv, *w, 3, D, rope_cos=cos, rope_sin=sin, pos_div=Sq, pos_mod=Tq)
    run = lambda c, s, pd, pm: E.qk_rmsnorm_(qkv.clone(), *w, 3, D, rope_cos=c, rope_sin=s, pos_div=pd, pos_mod=pm).view(-1, 3, 3, D)[:, :2]  # noqa: E731
    V.assert_legal("as is", run(cos, sin, Sq, Tq), ch)
    _rejects("position + 1", run(cos.roll(-1, 0), sin.roll(-1, 0), Sq, Tq), ch)
    pad = lambda t: torch.cat([t, t[:1].expand(Sq, D)])  # noqa: E731  (table rows for positions up to pos_mod = S)
    _rejects("pos_div and pos_mod swapped", run(pad(cos), pad(sin), Tq, Sq), ch)
    _rejects("pair sign flipped", run(cos, -sin, Sq, Tq), ch)
    _rejects("cos and sin swapped", run(sin, cos, Sq, Tq), ch)
    _rejects("truncated", V.round16(ch.v, dtype, mode="zero").to(dtype), ch)


@both
@pytest.mark.parametrize("D", [64, 72])
def test_qk_layernorm_chain_accepts_eager_and_rejects(D, dtype):
    qkv, wq, wk, _, _, _, _ = _qk_case(dtype, D)
    bq, bk = _rand(D, dtype=dtype, scale=0.1, seed=13), _rand(D, dtype=dtype, scale=0.1, seed=14)
    ch = R.qk_layernorm_chain(qkv, wq, bq, wk, bk, 3, D, eps=1e-5)
    R.assert_qk("eager", E.qk_layernorm_(qkv.clone(), wq, bq, wk, bk, 3, D, eps=1e-5), qkv, ch)
    _rejects("q and k parameters swapped", E.qk_layernorm_(qkv.clone(), wk, bk, wq, bq, 3, D, eps=1e-5).view(-1, 3, 3, D)[:, :2], ch)
    xf = qkv.float()[:, :2]
    g, b = torch.stack([wq, wk]).view(1, 2, 1, D).float(), torch.stack([bq, bk]).view(1, 2, 1, D).float()
    d = xf - xf.mean(-1, keepdim=True)
    bessel = (d * torch.rsqrt(d.pow(2).sum(-1, keepdim=True) / (D - 1) + 1e-5) * g + b).to(dtype)
    _rejects("variance over D - 1", bessel, ch)
    two = (d * torch.rsqrt(d.pow(2).mean(-1, keepdim=True) + 1e-5)).to(dtype) * g.to(dtype) + b.to(dtype)
    _rejects("rounded after every op", two, ch)
    whole = F.layer_norm(qkv.float()[:, :2].flatten(-2), (3 * D,)).view(-1, 2, 3, D)  # statistics over all heads
    _rejects("statistics across heads", (whole * g + b).to(dtype), ch)


@both
@pytest.mark.parametrize("D,half", [(72, 36), (72, 18), (96, 16), (72, 12)])
def test_qk_rope_halves_ref_equals_eager_and_rejects(D, half, dtype):
    qkv, _, _, _, _, Sq, Tq = _qk_case(dtype, D)
    rows = qkv.shape[0]
    ang = torch.arange(rows).view(rows, 1) * torch.linspace(0.05, 1.0, D).view(1, D)
    sign = torch.cat([-torch.ones(half), torch.ones(half)]).repeat(D // (2 * half))
    cos, sin = ang.cos().to(dtype).float(), (ang.sin().to(dtype).float() * sign)
    want = R.qk_rope_halves_ref(qkv, cos, sin, 3, D, half, 1, rows)
    V.assert_bit_exact("eager", E.qk_rope_halves_(qkv.clone(), cos, sin, 3, D, half, 1, rows), want)
    other = {36: 18, 18: 36, 16: 8, 12: 6}[half]
    _differs("partner from the wrong block", E.qk_rope_halves_(qkv.clone(), cos, sin, 3, D, other, 1, rows), want)
    _differs("position + 1", E.qk_rope_halves_(qkv.clone(), cos.roll(-1, 0), sin.roll(-1, 0), 3, D, half, 1, rows), want)
    t = qkv.float()[:, :2]
    partner = t.reshape(rows, 2, 3, D // (2 * half), 2, half).flip(4).reshape(rows, 2, 3, D)
    fused = torch.cat([(t * cos.view(rows, 1, 1, D) + partner * sin.view(rows, 1, 1, D)).to(dtype), qkv[:, 2:]], 1)
    _differs("products not rounded", fused, want)


# ---------------------------------------------------------------------------------------------------------------------
# depth-wise convolutions, kv_compress, patch_embed
# ---------------------------------------------------------------------------------------------------------------------
def _dw_case(dtype, ks, Bq=2, Tq=4, Hq=6, Wq=10, Cq=16):
    x = _hidden(Bq, Tq * Hq * Wq, Cq, dtype=dtype, seed=20)
    K = ks[0] * ks[1] * ks[2]
    taps = _rand(K, Cq, dtype=dtype, scale=0.3, seed=21)
    bias = _rand(Cq, dtype=dtype, scale=0.3, seed=22)
    return x, taps, bias, Bq, Tq, Hq, Wq


def _eager_dw(x, taps, bias, Bq, Tq, Hq, Wq, ks):
    """fp32 convolution, rounded; + bias, rounded; + x, rounded -- torch's CPU convolution adds the bias in fp32."""
    Cq = x.shape[-1]
    xi = x.reshape(Bq, Tq, Hq, Wq, Cq).permute(0, 4, 1, 2, 3)
    conv = F.conv3d(xi.float(), taps.float().t().reshape(Cq, 1, *ks), None, padding=tuple(k // 2 for k in ks), groups=Cq).to(x.dtype)
    return ((conv + bias.view(1, Cq, 1, 1, 1)) + xi).permute(0, 2, 3, 4, 1)


@both
@pytest.mark.parametrize("ks", [(3, 3, 3), (1, 3, 3), (3, 5, 5), (1, 5, 5), (3, 3, 5), (1, 3, 5), (3, 5, 3), (1, 5, 3)])
def test_dwconv_chain_accepts_eager(ks, dtype):
    x, taps, bias, *g = _dw_case(dtype, ks)
    V.assert_legal(f"dwconv {ks}", _eager_dw(x, taps, bias, *g, ks), R.dwconv_chain(x, taps, bias, *g, ks))
    x1, taps, bias, *g1 = _dw_case(dtype, ks, Tq=1, Hq=1, Wq=2)  # smaller than the kernel
    V.assert_legal(f"dwconv {ks} 1x1x2", _eager_dw(x1, taps, bias, *g1, ks), R.dwconv_chain(x1, taps, bias, *g1, ks))


@both
def test_rejects_dwconv_bugs(dtype):
    ks = (3, 3, 3)
    x, taps, bias, *g = _dw_case(dtype, ks)
    ch = R.dwconv_chain(x, taps, bias, *g, ks)
    got = _eager_dw(x, taps, bias, *g, ks)
    wm = taps.clone()
    wm[(1 * 3 + 1) * 3 + 0] = 0  # the tap at (t, h, w - 1)
    got[:, :, :, -1] = _eager_dw(x, wm, bias, *g, ks)[:, :, :, -1]
    _rejects("tap missing on the last column", got, ch)
    inner = torch.ones(got.shape[:4], dtype=torch.bool)
    inner[:, :, :, -1] = False
    assert V.check("other columns", got, ch, mask=inner)[0]
    Cq = x.shape[-1]
    xi = x.reshape(*g, Cq).permute(0, 4, 1, 2, 3)
    fused = F.conv3d(xi.float(), taps.float().t().reshape(Cq, 1, *ks), bias.float(), padding=1, groups=Cq).to(dtype) + xi
    _rejects("conv not rounded before the bias", fused.permute(0, 2, 3, 4, 1), ch)
    circ = F.conv3d(F.pad(xi.float(), (1, 1, 1, 1, 1, 1), mode="circular"), taps.float().t().reshape(Cq, 1, *ks), None, groups=Cq).to(dtype)
    _rejects("wrap-around padding", ((circ + bias.view(1, Cq, 1, 1, 1)) + xi).permute(0, 2, 3, 4, 1), ch)
    V.assert_bit_exact("shuffle order", EDS.dwconv_shuffle(x, torch.zeros_like(taps), torch.zeros_like(bias), *g, ks, (2, 2, 2)),
                       R.shuffle_rows(x.reshape(*g, Cq), *g, (2, 2, 2)).contiguous())


def _eager_ffn(h, taps, bias, BT, Hq, Wq, fuse_last=False):
    """out = out + module(x) per kernel size, each conv rounded before its bias; fuse_last: the 3x3 and 1x1 branches added in
    fp32 with one rounding."""
    Cq = h.shape[-1]
    xi = h.reshape(BT, Hq, Wq, Cq).permute(0, 3, 1, 2)
    c, o = [], 0
    for i, k in enumerate((5, 3, 1)):
        conv = F.conv2d(xi.float(), taps[o:o + k * k].float().t().reshape(Cq, 1, k, k), None, padding=k // 2, groups=Cq).to(h.dtype)
        c.append(conv + bias[i].view(1, Cq, 1, 1))
        o += k * k
    s = xi + c[0]
    out = (s.float() + c[1].float() + c[2].float()).to(h.dtype) if fuse_last else (s + c[1]) + c[2]
    return out.permute(0, 2, 3, 1)


@both
def test_dwconv_ffn_chain_accepts_eager_and_rejects(dtype):
    BT, Hq, Wq, Cq = 3, 9, 13, 16
    h = _hidden(BT, Hq, Wq, Cq, dtype=dtype, seed=23)
    taps, bias = _rand(35, Cq, dtype=dtype, scale=0.2, seed=24), _rand(3, Cq, dtype=dtype, scale=0.3, seed=25)
    ch = R.dwconv_ffn_chain(h, taps, bias, BT, Hq, Wq)
    V.assert_legal("ffn", _eager_ffn(h, taps, bias, BT, Hq, Wq).unsqueeze(1), ch)
    h1 = _hidden(2, 1, 3, Cq, dtype=dtype, seed=26)
    V.assert_legal("ffn 1x3", _eager_ffn(h1, taps, bias, 2, 1, 3).unsqueeze(1), R.dwconv_ffn_chain(h1, taps, bias, 2, 1, 3))
    sw = torch.cat([taps[:25], taps[25:34].flip(0), taps[34:]])
    _rejects("3x3 taps mirrored", _eager_ffn(h, sw, bias, BT, Hq, Wq).unsqueeze(1), ch)
    _rejects("biases of 5x5 and 3x3 swapped", _eager_ffn(h, taps, bias[[1, 0, 2]], BT, Hq, Wq).unsqueeze(1), ch)
    _rejects("no rounding between the last two adds", _eager_ffn(h, taps, bias, BT, Hq, Wq, fuse_last=True).unsqueeze(1), ch)


def _kvc_case(dtype, Cq=64):
    Bq, Tq, Hq, Wq = 2, 5, 5, 7
    x = _hidden(Bq, Tq, Hq, Wq, Cq, dtype=dtype, seed=30)
    x[:, 0] = _hidden(Bq, Hq, Wq, Cq, dtype=dtype, seed=31, offset=-1.0)  # frame 0 unlike the others
    ln_w = _rand(Cq, dtype=dtype, scale=0.2, offset=1.0, seed=33)
    ln_b = _rand(Cq, dtype=dtype, scale=0.1, seed=34)
    bias = _rand(Cq, dtype=dtype, scale=0.3, seed=35)
    return x, bias, ln_w, ln_b, Bq, Tq, Hq, Wq


def _eager_kvc(x, taps, bias, ln_w, ln_b, Bq, Tq, Hq, Wq, window, pad_t, round_conv, pad_frame=0, eps=1e-5):
    Cq = x.shape[-1]
    v = torch.cat([x[:, pad_frame:pad_frame + 1].expand(Bq, pad_t, Hq, Wq, Cq), x], 1) if pad_t else x
    xi = v.permute(0, 4, 1, 2, 3).float()
    w = taps.float().t().reshape(Cq, 1, *window)
    if round_conv:
        y = F.conv3d(xi, w, None, stride=window, groups=Cq).to(x.dtype) + bias.view(1, Cq, 1, 1, 1)
    else:
        y = F.conv3d(xi, w, bias.float(), stride=window, groups=Cq).to(x.dtype)
    return F.layer_norm(y.permute(0, 2, 3, 4, 1), (Cq,), ln_w, ln_b, eps)


KVC_WINDOWS = [((1, 2, 2), 0), ((1, 3, 3), 0), ((2, 1, 1), 0), ((2, 1, 1), 1), ((3, 1, 1), 2), ((4, 1, 1), 1)]


@both
@pytest.mark.parametrize("window,pad_t", KVC_WINDOWS)
def test_kv_compress_chain_accepts_eager(window, pad_t, dtype):
    x, bias, ln_w, ln_b, *g = _kvc_case(dtype)
    taps = _rand(window[0] * window[1] * window[2], x.shape[-1], dtype=dtype, scale=0.4, seed=32)
    for rc in (True, False):
        ch, _ = R.kv_compress_chain(x, taps, bias, ln_w, ln_b, *g, window, pad_t, 1e-5, rc)
        V.assert_legal(f"kv_compress {window} pad {pad_t} rc={int(rc)}", _eager_kvc(x, taps, bias, ln_w, ln_b, *g, window, pad_t, rc), ch)
    V.assert_legal("stand-in", EKV.kv_compress(x, taps, bias, ln_w, ln_b, *g, window, pad_t),
                   R.kv_compress_chain(x, taps, bias, ln_w, ln_b, *g, window, pad_t, 1e-5, False)[0])


@both
def test_rejects_kv_compress_bugs(dtype):
    x, bias, ln_w, ln_b, *g = _kvc_case(dtype)
    window, pad_t = (3, 1, 1), 2
    taps = _rand(3, x.shape[-1], dtype=dtype, scale=0.4, seed=32)
    for rc in (True, False):
        ch, y = R.kv_compress_chain(x, taps, bias, ln_w, ln_b, *g, window, pad_t, 1e-5, rc)
        st = _rejects("pad from frame 1", _eager_kvc(x, taps, bias, ln_w, ln_b, *g, window, pad_t, rc, pad_frame=1), ch)
        first = torch.zeros(ch.near.shape[:4], dtype=torch.bool)
        first[:, 0] = True
        assert st["bad"] > 0 and V.check("later windows", _eager_kvc(x, taps, bias, ln_w, ln_b, *g, window, pad_t, rc, pad_frame=1), ch, mask=~first)[0]
        _rejects("round_conv inverted", _eager_kvc(x, taps, bias, ln_w, ln_b, *g, window, pad_t, not rc), ch)
        small, nob = (x.float() * 0.002).to(dtype), torch.zeros_like(bias)  # small rows: eps is a visible part of var + eps
        _rejects("LayerNorm eps 1e-6", _eager_kvc(small, taps, nob, ln_w, ln_b, *g, window, pad_t, rc, eps=1e-6),
                 R.kv_compress_chain(small, taps, nob, ln_w, ln_b, *g, window, pad_t, 1e-5, rc)[0])
        _rejects("taps reversed", _eager_kvc(x, taps.flip(0), bias, ln_w, ln_b, *g, window, pad_t, rc), ch)


def _pe_case(dtype, Hq=9, Wq=15, Cq=64):
    z = _rand(2, 4, 2, Hq, Wq, dtype=dtype, offset=0.2, seed=40)
    w = _rand(Cq, 4, 1, 2, 2, dtype=dtype, scale=0.3, seed=41)
    bias = _rand(Cq, dtype=dtype, scale=0.2, seed=42)
    Sq = -(-Hq // 2) * -(-Wq // 2)
    pos = _rand(Sq, Cq, dtype=dtype, seed=43)
    return z, w, bias, pos


def _eager_pe(z, w, bias, pos, pad_value=0.0, fuse_bias=False):
    Bq, _, Tq, Hq, Wq = z.shape
    zp = F.pad(z.float(), (0, -Wq % 2, 0, -Hq % 2), value=pad_value)
    if fuse_bias:
        c = F.conv3d(zp, w.float(), bias.float(), stride=(1, 2, 2)).to(z.dtype)
    else:
        c = F.conv3d(zp, w.float(), None, stride=(1, 2, 2)).to(z.dtype) + bias.view(1, -1, 1, 1, 1)
    return c.flatten(3).permute(0, 2, 3, 1) + pos


@both
def test_patch_embed_chain_accepts_eager_and_rejects(dtype):
    for Hq, Wq in ((12, 16), (9, 15)):
        z, w, bias, pos = _pe_case(dtype, Hq, Wq)
        ch = R.patch_embed_chain(z, w, bias, pos, 2, 2)
        V.assert_legal(f"patch_embed {Hq}x{Wq}", _eager_pe(z, w, bias, pos), ch)
    _rejects("pad region not zero", _eager_pe(z, w, bias, pos, pad_value=1.0), ch)
    _rejects("bias inside the fp32 sum", _eager_pe(z, w, bias, pos, fuse_bias=True), ch)
    _rejects("position of the next patch", _eager_pe(z, w, bias, pos.roll(-1, 0)), ch)
    _rejects("taps in (dy, dx, c) order", _eager_pe(z, w.permute(0, 3, 4, 1, 2).reshape(w.shape), bias, pos), ch)
