"""The transformer-block kernels (csrc/elementwise.cu, csrc/dwconv.cu, csrc/patch_embed.cu) element by element against
float64, in bf16 and fp16, under the acceptance rule of tests/vae_fp64.py with the reference chains of tests/dit_fp64.py.

Arithmetic kernels are checked with assert_legal / check (every element inside the legal set of its chain; each check
prints eps, the bit-equal fraction, the largest error in ulps, the accepted flips with their distance to the midpoint, and
the count outside the legal set); kernels whose chain has one legal value, and all data movement, bit for bit.  Inputs look
like DiT hidden states: a DC offset and four channels x 20; the statistics tests add the (offset, sigma) grid of the
GroupNorm tests, a constant row and (fp16) values near the top of the range.  Every arithmetic kernel is launched twice
and the two results compared with torch.equal.

Which case reaches which template instance:
  ln_modulate_kernel<5, ., 3>   C <= 1280          C = 8 (one lane), 64, 288, 1152, 1280
  ln_modulate_kernel<8, ., 2>   C <= 2048          C = 1288, 1920, 2048
  ln_modulate_kernel<9, ., 2>   C <= 2304          C = 2056, 2304
  ln_modulate_kernel<12, ., 1>  C <= 3072          C = 2312, 3072
  qk_rmsnorm_kernel<64>, <72>; qk_layernorm_kernel<64>, <72>      D = 64, 72 (every other D is refused: D = 80)
  qk_rope_halves_kernel (one instance)             (D, half) = (72, 36), (72, 18), (96, 16), (72, 12), (64, 32), (64, 16)
  dwconv_shuffle_kernel<kt, kh, kw>                all eight of kt in {1, 3} x kh, kw in {3, 5}
  kv_compress_kernel<5>  C <= 1280                 C = 64, 1152, 1280
  kv_compress_kernel<12> C <= 3072                 C = 1288, 3072
  gate_residual, residual_add, gate_residual_unshuffle, modulation_table, dwconv_ffn, patch_embed: one instance each."""
import pytest
import torch

from tests import dit_fp64 as R
from tests import vae_fp64 as V
from tests.test_vae_kernels_fp64_gpu import OFFSET_SIGMA
from videosys_b200 import kernels
from videosys_b200._lib import VsbError

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]
both = pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
WIDTHS = [8, 64, 288, 1152, 1280, 1288, 1920, 2048, 2056, 2304, 2312, 3072]
ROW_PAIRS = [(0, 1), (3, 4), (1, 0)]  # (shift, scale) rows the models pass


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _rand(*shape, dtype, scale=1.0, offset=0.0, seed=0):
    return (offset + scale * torch.randn(*shape, generator=_gen(seed))).to(dtype).to(DEV)


def _hidden(*shape, dtype, seed, offset=0.3):
    """DiT-like hidden states, channels last: a DC offset and four massive channels (x 20)."""
    z = offset + torch.randn(*shape, generator=_gen(seed))
    z[..., 3:7] *= 20
    return z.to(dtype).to(DEV)


def _masks(B, T):
    """Name -> uint8 [B, T] (None: no mask): all frames on / off, and the first / last frame of the first / last sample off."""
    ones = torch.ones(B, T, dtype=torch.uint8)
    edge = ones.clone()
    edge[0, 0] = edge[-1, -1] = 0
    edge2 = ones.clone()
    edge2[0, -1] = edge2[-1, 0] = 0
    return {"none": None, "ones": ones.to(DEV), "zeros": (0 * ones).to(DEV), "first/last off": edge.to(DEV), "last/first off": edge2.to(DEV)}


def _guarded(rows, C, dtype):
    """A NaN-filled buffer and its interior [rows, C] view (16-byte aligned for every C % 8 == 0)."""
    buf = torch.full((rows + 2, C), float("nan"), dtype=dtype, device=DEV)
    return buf, buf[1:-1]


def _guards_intact(what, buf):
    assert bool(torch.isnan(buf[0].float()).all() and torch.isnan(buf[-1].float()).all()), f"{what}: wrote outside its output"


# =====================================================================================================================
# ln_modulate / ln_modulate_affine
# =====================================================================================================================
def _ln_run(what, x, mod, mask, pair, B, T, S, eps, gamma, beta):
    C = x.shape[-1]
    buf, out = _guarded(B * T * S, C, x.dtype)
    kernels.ln_modulate(x, mod, mask, *pair, B, T, S, out=out, eps=eps, gamma=gamma, beta=beta)
    _guards_intact(what, buf)
    assert torch.equal(out, kernels.ln_modulate(x, mod, mask, *pair, B, T, S, eps=eps, gamma=gamma, beta=beta).view_as(out)), f"{what}: two launches differ"
    ch = R.ln_modulate_chain(x, mod, mask, *pair, B, T, S, eps=eps, gamma=gamma, beta=beta)
    ok = V.check(what, out.view(B, T, S, C), ch)[0]  # the eps it prints is the last rounding point's: zero
    print(f"    {100 * float((ch.lo != ch.hi).double().mean()):.4f} % of the elements have more than one legal value")
    return ok


@both
@pytest.mark.parametrize("C", WIDTHS)
def test_ln_modulate_fp64(C, dtype):
    gamma = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=3)
    beta = _rand(C, dtype=dtype, scale=0.1, seed=4)
    # (B, T, S): one row; fewer rows than one CTA has warps; some hundred; at the top width of every instance enough that
    # every warp of the capped grid takes several rows of the grid-stride loop
    shapes = [(1, 1, 1), (1, 7, 1), (2, 3, 50)] + ([(2, 4, 3200)] if C in (1280, 2048, 2304, 3072) else [])
    failed, k = [], 0
    for B, T, S in shapes:
        x = _hidden(B * T * S, C, dtype=dtype, seed=1)
        mod = _rand(2, B, 6, C, dtype=dtype, scale=0.5, seed=2)
        masks = _masks(B, T)
        for mname in (masks if S == 50 else ("none", "first/last off")):
            for affine in (False, True):
                pair, eps = ROW_PAIRS[k % 3], (1e-6, 1e-5)[(k // 3) % 2]
                k += 1
                what = f"ln_modulate{'_affine' if affine else ''} {dtype} C={C} [{B},{T},{S}] mask={mname} rows={pair} eps={eps}"
                if not _ln_run(what, x, mod, masks[mname], pair, B, T, S, eps, gamma if affine else None, beta if affine else None):
                    failed.append(what)
    assert not failed, failed


@both
@pytest.mark.parametrize("C", [64, 1152, 3072])
def test_ln_modulate_statistics_fp64(C, dtype):
    """LayerNorm statistics where fp32 statistics go wrong: a large offset with a small spread, massive channels, values
    near the top of fp16, for both eps the models use."""
    B, T, S = 2, 2, 16
    mod = _rand(2, B, 6, C, dtype=dtype, scale=0.5, seed=2)
    gamma, beta = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=3), _rand(C, dtype=dtype, scale=0.1, seed=4)
    grid = OFFSET_SIGMA + [(3e4, 5e3)] + ([(-5e4, 3e3)] if dtype == torch.float16 else [])
    failed = []
    for i, (offset, sigma) in enumerate(grid):
        x = _rand(B * T * S, C, dtype=dtype, scale=sigma, offset=offset, seed=20 + i)
        for eps in (1e-6, 1e-5):
            for gb in ((None, None), (gamma, beta)):
                what = f"ln_modulate{'_affine' if gb[0] is not None else ''} {dtype} C={C} offset={offset} sigma={sigma} eps={eps}"
                if not _ln_run(what, x, mod, None, (0, 1), B, T, S, eps, *gb):
                    failed.append(what)
    assert not failed, failed


@both
@pytest.mark.parametrize("C", [8, 1152, 3072])
def test_ln_modulate_constant_row_exact(C, dtype):
    """A constant row: every fp32 partial sum k * x is exact, the mean is x and the variance zero, so n is exactly zero
    (rstd = eps^-1/2 multiplies it) whatever the summation order, and the output is r(r(beta * g) + shift)."""
    B, T, S = 2, 3, 5
    x = torch.tensor([10.0, -0.75, 3.0, 0.0, 1e-3, 200.0], dtype=dtype, device=DEV).repeat(5).view(-1, 1).expand(B * T * S, C).contiguous()
    mod = _rand(2, B, 6, C, dtype=dtype, scale=0.5, seed=2)
    gamma, beta = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=3), _rand(C, dtype=dtype, scale=0.1, seed=4)
    mask = _masks(B, T)["first/last off"]
    g = V.round16(1.0 + R.mod_row(mod, mask, 1, B, T), dtype)
    sh = R.mod_row(mod, mask, 0, B, T)
    for eps in (1e-6, 1e-5):
        for gb, n in (((None, None), torch.zeros(C, dtype=torch.float64, device=DEV)), ((gamma, beta), beta.double())):
            want = V.round16(V.round16(n * g, dtype) + sh, dtype).expand(B, T, S, C).to(dtype)
            got = kernels.ln_modulate(x, mod, mask, 0, 1, B, T, S, eps=eps, gamma=gb[0], beta=gb[1])
            V.assert_bit_exact(f"ln_modulate constant rows {dtype} C={C} eps={eps} affine={gb[0] is not None}", got.view(B, T, S, C), want.contiguous())
            assert R.check("the chain accepts it", got.view(B, T, S, C), R.ln_modulate_chain(x, mod, mask, 0, 1, B, T, S, eps, *gb))[0]


@both
@pytest.mark.parametrize("C", [3080, 12, 4])
def test_ln_modulate_refuses_unsupported_width(C, dtype):
    """Argument checks that return before any launch: wider than the widest instance, or not a whole number of vectors."""
    x = _rand(4, C, dtype=dtype)
    mod = _rand(2, 1, 6, C, dtype=dtype)
    g = _rand(C, dtype=dtype)
    n0 = kernels.launch_count()
    with pytest.raises(VsbError, match=r"status -2"):
        kernels.ln_modulate(x, mod, None, 0, 1, 1, 1, 4)
    with pytest.raises(VsbError, match=r"status -2"):
        kernels.ln_modulate(x, mod, None, 0, 1, 1, 1, 4, gamma=g, beta=g)
    assert kernels.launch_count() == n0


# =====================================================================================================================
# modulation_table, gate_residual, residual_add, gate_residual_unshuffle: one legal value per element
# =====================================================================================================================
@both
@pytest.mark.parametrize("rows", [6, 2])
def test_modulation_table_exact(rows, dtype):
    for B, C in ((1, 8), (2, 1152), (3, 3072)):
        table = _rand(rows, C, dtype=dtype, seed=7)
        t, t0 = _hidden(B, rows * C, dtype=dtype, seed=8), _hidden(B, rows * C, dtype=dtype, seed=9, offset=-0.5)
        for tt0 in (t0, None):
            V.assert_bit_exact(f"modulation_table {dtype} rows={rows} B={B} C={C} t0={tt0 is not None}",
                               kernels.modulation_table(table, t, tt0), R.modulation_table_ref(table, t, tt0))


@both
@pytest.mark.parametrize("C", WIDTHS)
def test_gate_residual_and_residual_add_exact(C, dtype):
    for B, T, S in ((1, 1, 1), (2, 3, 50), (2, 4, 700)):
        x, y = _hidden(B * T * S, C, dtype=dtype, seed=1), _hidden(B * T * S, C, dtype=dtype, seed=5, offset=-0.2)
        mod = _rand(2, B, 6, C, dtype=dtype, scale=0.5, seed=2)
        for i, (mname, mask) in enumerate(_masks(B, T).items()):
            gate_row = (2, 5)[i % 2]
            what = f"gate_residual {dtype} C={C} [{B},{T},{S}] mask={mname} row={gate_row}"
            cache, want = R.gate_residual_ref(x, y, mod, mask, gate_row, B, T, S)
            buf, out = _guarded(B * T * S, C, dtype)
            cbuf, cout = _guarded(B * T * S, C, dtype)
            kernels.gate_residual(x, y, mod, mask, gate_row, B, T, S, out=out, cache_out=cout)
            _guards_intact(what, buf), _guards_intact(what + " cache", cbuf)
            V.assert_bit_exact(what, out, want)
            V.assert_bit_exact(what + " cache_out", cout, cache)
            V.assert_bit_exact(what + " no cache", kernels.gate_residual(x, y, mod, mask, gate_row, B, T, S), want)
            xi = x.clone()
            kernels.gate_residual(xi, y, mod, mask, gate_row, B, T, S, out=xi)  # in place, as the models call it
            V.assert_bit_exact(what + " in place", xi, want)
        V.assert_bit_exact(f"residual_add {dtype} C={C} rows={B * T * S}", kernels.residual_add(x, y), R.residual_add_ref(x, y))
        xi = x.clone()
        V.assert_bit_exact(f"residual_add {dtype} C={C} in place", kernels.residual_add(xi, y, out=xi), R.residual_add_ref(x, y))


@both
@pytest.mark.parametrize("down", [(2, 2, 2), (1, 2, 2), (2, 1, 3), (1, 1, 1)])
def test_gate_residual_unshuffle_exact(down, dtype):
    for B, T, H, W, C in ((2, 4, 6, 12, 2304), (1, 2, 2, 6, 8), (3, 2, 4, 6, 264)):
        N = T * H * W
        x = _hidden(B, N, C, dtype=dtype, seed=1)
        mod = _rand(2, B, 6, C, dtype=dtype, scale=0.5, seed=2)
        # every row of y carries a code of its own index, far more than an ulp apart: a wrong gather cannot hide
        code = ((torch.arange(B * N) * 37) % 255 - 127).view(-1, 1).float()
        y = (code + torch.randn(B * N, C, generator=_gen(3))).to(dtype).to(DEV).view(B * down[0] * down[1] * down[2], -1, C)
        want = R.gate_residual_unshuffle_ref(x, y, mod, 2, B, T, H, W, down)
        what = f"gate_residual_unshuffle {dtype} [{B},{T},{H},{W},{C}] down={down}"
        V.assert_bit_exact(what, kernels.gate_residual_unshuffle(x, y, mod, 2, B, T, H, W, down), want)
        xi = x.clone()
        V.assert_bit_exact(what + " in place", kernels.gate_residual_unshuffle(xi, y, mod, 2, B, T, H, W, down, out=xi), want)


# =====================================================================================================================
# q / k normalisation and RoPE on the packed qkv buffer
# =====================================================================================================================
def _qkv(rows, H, D, dtype, seed=10):
    """Heads with a DC offset (head 0) and with one channel x 50 (the last head)."""
    z = 0.4 + torch.randn(rows, 3, H, D, generator=_gen(seed))
    z[:, :, 0] += 2
    z[:, :, -1, 5] *= 50
    return z.to(dtype).to(DEV)


def _rope_tables(T, D):
    ang = torch.arange(T).view(T, 1) * (10000.0 ** (-torch.arange(0, D, 2) / D)).repeat_interleave(2).view(1, D)
    return ang.cos().contiguous().to(DEV), ang.sin().contiguous().to(DEV)


# 1 row; 77; 101 rows leave idle tail groups in the last warp for every H (2 * H * 101 is no multiple of 12 or 16 when H is
# odd; for H = 16, 30 the tail is in the unrolled U = 4 slots); 1500 rows put several trips of the grid-stride loop on
# the layernorm kernel
QK_ROWS = [1, 77, 101, 1500]


def _twice(fn, qkv):
    a, b = fn(qkv.clone()), fn(qkv.clone())
    assert torch.equal(a, b), "two launches differ"
    return a


@both
@pytest.mark.parametrize("H", [1, 3, 16, 30])
@pytest.mark.parametrize("D", [64, 72])
def test_qk_rmsnorm_and_rope_fp64(D, H, dtype):
    wq = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=11)
    wk = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=12)
    S, T = 5, 7
    cos, sin = _rope_tables(T, D)
    failed = []
    for rows in QK_ROWS:
        qkv = _qkv(rows, H, D, dtype)
        variants = {"norm": (wq, wk, {}),
                    "norm+rope": (wq, wk, dict(rope_cos=cos, rope_sin=sin, pos_div=S, pos_mod=T)),  # rows no multiple of S * T
                    "rope only": (None, None, dict(rope_cos=cos, rope_sin=sin, pos_div=S, pos_mod=T)),
                    "norm+rope T=1": (wq, wk, dict(rope_cos=cos[3:4].contiguous(), rope_sin=sin[3:4].contiguous(), pos_div=S, pos_mod=1)),
                    "norm eps=1e-5": (wq, wk, dict(eps=1e-5))}
        for name, (a, b, kw) in variants.items():
            what = f"qk_rmsnorm_ {name} {dtype} rows={rows} H={H} D={D}"
            got = _twice(lambda t: kernels.qk_rmsnorm_(t, a, b, H, D, **kw), qkv)
            try:
                R.assert_qk(what, got, qkv, R.qk_rmsnorm_chain(qkv, a, b, H, D, **kw))
            except AssertionError as e:
                failed.append(f"{what}: {e}")
    assert not failed, failed


@both
@pytest.mark.parametrize("H", [1, 3, 16, 30])
@pytest.mark.parametrize("D", [64, 72])
def test_qk_layernorm_fp64(D, H, dtype):
    wq, wk = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=11), _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=12)
    bq, bk = _rand(D, dtype=dtype, scale=0.1, seed=13), _rand(D, dtype=dtype, scale=0.1, seed=14)
    failed = []
    for rows in QK_ROWS:
        for eps in (1e-6, 1e-5):
            qkv = _qkv(rows, H, D, dtype)
            what = f"qk_layernorm_ {dtype} rows={rows} H={H} D={D} eps={eps}"
            got = _twice(lambda t: kernels.qk_layernorm_(t, wq, bq, wk, bk, H, D, eps=eps), qkv)
            try:
                R.assert_qk(what, got, qkv, R.qk_layernorm_chain(qkv, wq, bq, wk, bk, H, D, eps))
            except AssertionError as e:
                failed.append(f"{what}: {e}")
    assert not failed, failed


@both
@pytest.mark.parametrize("D", [64, 72])
def test_qk_norm_statistics_fp64(D, dtype):
    """Per-head statistics on the (offset, sigma) grid, and constant heads (LayerNorm: exactly the bias)."""
    H, rows = 3, 50
    wq, wk = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=11), _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=12)
    bq, bk = _rand(D, dtype=dtype, scale=0.1, seed=13), _rand(D, dtype=dtype, scale=0.1, seed=14)
    failed = []
    for i, (offset, sigma) in enumerate(OFFSET_SIGMA + [(1e-3, 1e-3), (0, 0), (7, 0)]):
        qkv = _rand(rows, 3, H, D, dtype=dtype, scale=sigma, offset=offset, seed=30 + i)
        for name, fn, ch in (("qk_rmsnorm_", lambda t: kernels.qk_rmsnorm_(t, wq, wk, H, D), R.qk_rmsnorm_chain(qkv, wq, wk, H, D)),
                             ("qk_layernorm_", lambda t: kernels.qk_layernorm_(t, wq, bq, wk, bk, H, D, eps=1e-5),
                              R.qk_layernorm_chain(qkv, wq, bq, wk, bk, H, D, 1e-5))):
            what = f"{name} {dtype} D={D} offset={offset} sigma={sigma}"
            got = fn(qkv.clone())
            try:
                R.assert_qk(what, got, qkv, ch)
                if sigma == 0 and name == "qk_layernorm_":
                    want = torch.stack([bq, bk]).view(1, 2, 1, D).expand(rows, 2, H, D).contiguous()
                    V.assert_bit_exact(what + " constant heads give the bias", got.view(rows, 3, H, D)[:, :2].contiguous(), want)
            except AssertionError as e:
                failed.append(f"{what}: {e}")
    assert not failed, failed


@both
@pytest.mark.parametrize("D,half", [(72, 36), (72, 18), (96, 16), (72, 12), (64, 32), (64, 16)])
def test_qk_rope_halves_exact(D, half, dtype):
    """RoPE1D (half = D / 2), RoPE2D (D / 4) and RoPE3D (D / 6) of Open-Sora-Plan, tables of 16-bit values."""
    for H, rows, pos_div, pos_mod in ((1, 1, 1, 1), (3, 77, 1, 77), (16, 101, 5, 7), (24, 1500, 1, 1500)):
        qkv = _qkv(rows, H, D, dtype)
        ang = torch.arange(pos_mod).view(-1, 1) * torch.linspace(0.05, 1.0, D).view(1, D)
        sign = torch.cat([-torch.ones(half), torch.ones(half)]).repeat(D // (2 * half))
        cos, sin = ang.cos().to(dtype).float().to(DEV), (ang.sin().to(dtype).float() * sign).to(DEV)
        got = _twice(lambda t: kernels.qk_rope_halves_(t, cos, sin, H, D, half, pos_div, pos_mod), qkv)
        V.assert_bit_exact(f"qk_rope_halves_ {dtype} D={D} half={half} H={H} rows={rows} pos=(r // {pos_div}) % {pos_mod}",
                           got, R.qk_rope_halves_ref(qkv, cos, sin, H, D, half, pos_div, pos_mod))


@both
def test_qk_kernels_refuse_other_head_dims(dtype):
    D, H = 80, 2
    qkv, w = _qkv(4, H, D, dtype), _rand(D, dtype=dtype)
    n0 = kernels.launch_count()
    with pytest.raises(VsbError, match=r"status -2"):
        kernels.qk_rmsnorm_(qkv, w, w, H, D)
    with pytest.raises(VsbError, match=r"status -2"):
        kernels.qk_layernorm_(qkv, w, w, w, w, H, D)
    with pytest.raises(VsbError, match=r"status -2"):
        kernels.qk_rope_halves_(qkv, *_rope_tables(4, D), H, D, 24)  # 80 is no whole number of 48-channel blocks
    assert kernels.launch_count() == n0


# =====================================================================================================================
# depth-wise convolutions
# =====================================================================================================================
def _regions(B, T, H, W):
    """Border pixels, seam pixels of the 8-row x 4-column thread tile (not on the border), and the interior."""
    y = torch.arange(H, device=DEV).view(H, 1)
    x = torch.arange(W, device=DEV).view(1, W)
    border = (y == 0) | (y == H - 1) | (x == 0) | (x == W - 1)
    seam = ((x % 4 == 0) | (x % 4 == 3) | (y % 8 == 0) | (y % 8 == 7)) & ~border
    interior = ~border & ~seam
    return {k: m.expand(B, T, H, W) for k, m in (("border", border), ("seam", seam), ("interior", interior))}


KSIZES = [(3, 3, 3), (1, 3, 3), (3, 5, 5), (1, 5, 5), (3, 3, 5), (1, 3, 5), (3, 5, 3), (1, 5, 3)]
# (B, T, H, W, C, down): the released width with edge tiles; one pixel; smaller than the kernel; H, W no multiple of the
# tile and a second channel slice with one live lane; an asymmetric regrouping
DW_SHAPES = [(1, 4, 6, 10, 2304, (2, 2, 2)), (2, 1, 1, 1, 64, (1, 1, 1)), (1, 2, 2, 3, 8, (2, 1, 3)),
             (2, 2, 9, 14, 264, (1, 3, 7)), (1, 3, 17, 21, 512, (3, 1, 1))]


@both
@pytest.mark.parametrize("ks", KSIZES)
def test_dwconv_shuffle_fp64(ks, dtype):
    failed = []
    for B, T, H, W, C, down in DW_SHAPES:
        x = _hidden(B, T * H * W, C, dtype=dtype, seed=20)
        taps = _rand(ks[0] * ks[1] * ks[2], C, dtype=dtype, scale=0.3, seed=21)
        bias = _rand(C, dtype=dtype, scale=0.3, seed=22)
        got = kernels.dwconv_shuffle(x, taps, bias, B, T, H, W, ks, down)
        assert torch.equal(got, kernels.dwconv_shuffle(x, taps, bias, B, T, H, W, ks, down))
        nat = got.reshape(-1, C)[R.unshuffle_index(B, T, H, W, down, DEV)].view(B, T, H, W, C)
        ch = R.dwconv_chain(x, taps, bias, B, T, H, W, ks)
        for where, m in _regions(B, T, H, W).items():
            what = f"dwconv_shuffle {dtype} k={ks} [{B},{T},{H},{W},{C}] down={down} {where}"
            if bool(m.any()) and not V.check(what, nat, ch, mask=m)[0]:
                failed.append(what)
        # the store order alone: zero taps and bias leave r(0 + x) = x, every row moved to its sub-grid place
        z = kernels.dwconv_shuffle(x, torch.zeros_like(taps), torch.zeros_like(bias), B, T, H, W, ks, down)
        V.assert_bit_exact(f"dwconv_shuffle {dtype} k={ks} [{B},{T},{H},{W},{C}] down={down} order",
                           z, R.shuffle_rows(x.view(B, T, H, W, C), B, T, H, W, down).contiguous())
    assert not failed, failed


@both
def test_dwconv_ffn_fp64(dtype):
    failed = []
    for BT, H, W, C in ((2, 6, 10, 4608), (1, 1, 1, 64), (2, 1, 3, 128), (3, 9, 13, 264), (2, 30, 41, 512)):
        h = _hidden(BT, H, W, C, dtype=dtype, seed=23)
        taps, bias = _rand(35, C, dtype=dtype, scale=0.2, seed=24), _rand(3, C, dtype=dtype, scale=0.3, seed=25)
        got = kernels.dwconv_ffn(h, taps, bias, BT, H, W)
        assert torch.equal(got, kernels.dwconv_ffn(h, taps, bias, BT, H, W))
        ch = R.dwconv_ffn_chain(h, taps, bias, BT, H, W)
        for where, m in _regions(BT, 1, H, W).items():
            what = f"dwconv_ffn {dtype} [{BT},{H},{W},{C}] {where}"
            if bool(m.any()) and not V.check(what, got.view(BT, 1, H, W, C), ch, mask=m)[0]:
                failed.append(what)
    assert not failed, failed


# =====================================================================================================================
# kv_compress
# =====================================================================================================================
# (window, pad_t, T, H, W): spatial 2 and 3 on odd grids (last row / column unread), temporal with every pad
KVC_CASES = [((1, 2, 2), 0, 3, 7, 9), ((1, 3, 3), 0, 2, 7, 11), ((2, 1, 1), 0, 7, 5, 1), ((2, 1, 1), 1, 7, 5, 1),
             ((3, 1, 1), 2, 8, 3, 2), ((4, 1, 1), 1, 9, 6, 1), ((1, 2, 2), 0, 2, 40, 60)]


@both
@pytest.mark.parametrize("C", [64, 1152, 1280, 1288, 3072])
def test_kv_compress_fp64(C, dtype):
    B = 2
    ln_w, ln_b = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=33), _rand(C, dtype=dtype, scale=0.1, seed=34)
    bias = _rand(C, dtype=dtype, scale=0.3, seed=35)
    failed = []
    for window, pad_t, T, H, W in KVC_CASES:
        x = _hidden(B, T, H, W, C, dtype=dtype, seed=30)
        x[:, 0] = _hidden(B, H, W, C, dtype=dtype, seed=31, offset=-1.0)  # frame 0 unlike the others: the pad source shows
        taps = _rand(window[0] * window[1] * window[2], C, dtype=dtype, scale=0.4, seed=32)
        for rc in (True, False):
            for eps in (1e-5, 1e-6):
                what = f"kv_compress {dtype} C={C} [{B},{T},{H},{W}] window={window} pad_t={pad_t} round_conv={int(rc)} eps={eps}"
                got = kernels.kv_compress(x, taps, bias, ln_w, ln_b, B, T, H, W, window, pad_t, eps, rc)
                assert torch.equal(got, kernels.kv_compress(x, taps, bias, ln_w, ln_b, B, T, H, W, window, pad_t, eps, rc)), what
                ch, y = R.kv_compress_chain(x, taps, bias, ln_w, ln_b, B, T, H, W, window, pad_t, eps, rc)
                print(f"    conv rounding point: {int((y.lo != y.hi).sum())} of {y.near.numel()} elements with two legal values")
                if not V.check(what, got, ch)[0]:
                    failed.append(what)
    assert not failed, failed


@both
@pytest.mark.parametrize("C", [64, 1152, 3072])
def test_kv_compress_layernorm_statistics_fp64(C, dtype):
    """The LayerNorm inside kv_compress on the (offset, sigma) grid: a (1, 1, 1) window with a unit tap and no bias makes
    y = x exactly, so the statistics are those of a chosen row."""
    B, T, H, W = 1, 2, 4, 4
    ln_w, ln_b = _rand(C, dtype=dtype, scale=0.2, offset=1.0, seed=33), _rand(C, dtype=dtype, scale=0.1, seed=34)
    one, zero = torch.ones(1, C, dtype=dtype, device=DEV), torch.zeros(C, dtype=dtype, device=DEV)
    failed = []
    for i, (offset, sigma) in enumerate(OFFSET_SIGMA + [(0, 0), (7, 0)]):
        x = _rand(B, T, H, W, C, dtype=dtype, scale=sigma, offset=offset, seed=40 + i)
        if sigma:
            x[..., 3:7] *= 20
        for rc in (True, False):
            what = f"kv_compress LayerNorm {dtype} C={C} offset={offset} sigma={sigma} round_conv={int(rc)}"
            got = kernels.kv_compress(x, one, zero, ln_w, ln_b, B, T, H, W, (1, 1, 1), 0, 1e-5, rc)
            ch, y = R.kv_compress_chain(x, one, zero, ln_w, ln_b, B, T, H, W, (1, 1, 1), 0, 1e-5, rc)
            assert torch.equal(y.lo, y.hi) and torch.equal(y.near, x.double())
            if not V.check(what, got, ch)[0]:
                failed.append(what)
            if not sigma:  # constant rows: exactly the LayerNorm bias
                V.assert_bit_exact(what + " constant rows give ln_b", got, ln_b.expand_as(got).contiguous())
    assert not failed, failed


# =====================================================================================================================
# patch_embed
# =====================================================================================================================
@both
@pytest.mark.parametrize("B,Cin,T,H,W,C,ph,pw", [(2, 4, 3, 12, 16, 1152, 2, 2),   # exact patch grid
                                                   (1, 4, 2, 9, 15, 288, 2, 2),     # H, W no multiples of the patch: zero pad
                                                   (2, 4, 15, 30, 53, 1152, 2, 2),  # OpenSora 240p latent
                                                   (1, 16, 2, 6, 10, 64, 1, 1),     # 16 channels, 1 x 1 patch
                                                   (1, 4, 1, 1, 1, 8, 2, 2)])       # one patch, three of its four pixels padding
def test_patch_embed_fp64(B, Cin, T, H, W, C, ph, pw, dtype):
    z = _rand(B, Cin, T, H, W, dtype=dtype, offset=0.2, seed=40)
    z[:, 1] *= 8  # one latent channel larger than the others
    w = _rand(C, Cin, 1, ph, pw, dtype=dtype, scale=0.3, seed=41)
    bias = _rand(C, dtype=dtype, scale=0.2, seed=42)
    S = -(-H // ph) * -(-W // pw)
    pos = _rand(S, C, dtype=dtype, seed=43)
    what = f"patch_embed {dtype} [{B},{Cin},{T},{H},{W}] -> {C}"
    got = kernels.patch_embed(z, w, bias, pos, ph, pw)
    assert got is not None and got.shape == (B, T, S, C)
    assert torch.equal(got, kernels.patch_embed(z, w, bias, pos, ph, pw))
    V.assert_legal(what, got, R.patch_embed_chain(z, w, bias, pos, ph, pw))
    V.assert_legal(what + " no bias, no pos", kernels.patch_embed(z, w, None, None, ph, pw), R.patch_embed_chain(z, w, None, None, ph, pw))
    # the rank-local form: each rank's patch columns bit-equal to the full result, columns past the grid zero
    world = 3
    Sl = -(-S // world)
    full = torch.cat([got, torch.zeros(B, T, world * Sl - S, C, dtype=dtype, device=DEV)], 2)
    for r in range(world):
        part = kernels.patch_embed(z, w, bias, pos, ph, pw, s0=r * Sl, s_local=Sl)
        V.assert_bit_exact(f"{what} rank {r} of {world}", part, full[:, :, r * Sl:(r + 1) * Sl].contiguous())
