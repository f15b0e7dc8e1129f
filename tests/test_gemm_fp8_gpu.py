"""The e4m3 GEMM entries (vsb_gemm_fp8_bias_act / _residual, gemm_wide_kernel<fp8, .> in csrc/gemm_wgmma.cu) element by
element against float64, and the quantization kernels (vsb_quant_rows_fp8, vsb_ln_modulate_fp8) bit for bit against the
rule's torch restatement (tests/fp8_rule.py).

The reference of the GEMM is the float64 product of the dequantized operands, qa sa . qw sw = (qa . qw) sa sw exactly
(e4m3 codes times fp32 scales are exact in float64), and from y on the chains of tests/gemm_attn_fp64.py.  eps of y:

  acc   The products of two e4m3 values are exact in fp32.  The kernel sums each 128-element k-block on the tensor cores
        into a fresh fragment, four k32 steps, and adds the fragment to fp32 registers.  Inside a k-block the tensor core
        keeps a reduced-precision running sum (DeepSeek-V3 reports about 14 significant bits on Hopper); step s of block b
        is bounded by U_TC (|C_b,s-1| + sum_step |p|), U_TC = 2^-12, where C_b,s is the float64 partial sum of the block
        after step s (restarting at 0 in every block) and sum_step |p| the magnitudes of the step's 32 products, which
        the alignment of the addends can truncate.  The fp32 add of each block's fragment rounds by U32 |S_b|, S_b the
        float64 sum of blocks 0..b.  (U_TC = 2^-13, the reported 14 bits, left 2 of 2.95 million elements of a
        2561 x 1152 x 1152 product on an H100 outside the bound: the hardware's alignment of the addends costs up to one
        more bit.)
            eps_acc = U_TC sum_b sum_s (|C_b,s-1| + sum_step |p|) + U32 sum_b |S_b|
  y     t = fp32(acc sa) and y = fmaf(t, sw, bias): eps = eps_acc sa sw + U32 |acc sa sw| + U32 |y|.

Without the promotion the running sum of the whole K would carry the same 14 bits: the term U_TC sum |C_s| would run over
the partial sums of all K / 32 steps instead of those inside a block.  Where the products share a sign (a GELU output
against weights with a positive mean) the whole-K partial sums grow linearly, and at K = 4608 that sum is about 29 times
the per-block one: test_gemm_fp8_promotion_bound holds the kernel to the promoted bound there."""
import pytest
import torch

from tests import fp8_rule
from tests import gemm_attn_fp64 as G
from tests.test_dit_kernels_fp64_gpu import _masks
from tests.test_gemm_attn_kernels_fp64_gpu import DEV, DTYPES, IDS, _check, _guarded, _guards_intact, _hidden, _rand
from tests.vae_fp64 import U32, Chain
from videosys_b200 import _lib, kernels

pytestmark = pytest.mark.gpu
both = pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
U_TC = 2.0**-12  # relative precision of the tensor core's running sum of e4m3 products inside a k-block


def _acc_eps(qa, qw, block=128, step=32):
    """(float64 qa . qw^T, eps_acc of the module docstring) of codes qa [M, K], qw [N, K]."""
    ad, wd = qa.double(), qw.double()
    M, K = ad.shape
    acc = ad @ wd.T
    eps = U_TC * (ad.abs() @ wd.abs().T)
    S = torch.zeros_like(acc)
    for b0 in range(0, K, block):
        c = torch.zeros_like(acc)
        for k0 in range(b0, min(b0 + block, K), step):
            eps += U_TC * c.abs()
            c += ad[:, k0:k0 + step] @ wd[:, k0:k0 + step].T
        S += c
        eps += U32 * S.abs()
    return acc, eps


def fp8_linear_chain(qa, sa, qw, sw, bias, dtype):
    acc, e = _acc_eps(qa.float(), qw.float())
    s = sa.double()[:, None] * sw.double()[None, :]
    v = acc * s
    if bias is not None:
        v = v + bias.double()
    return Chain.start(v, e * s + U32 * (acc * s).abs() + U32 * v.abs(), dtype)


def fp8_chain(qa, sa, qw, sw, bias, act, dtype):
    y = fp8_linear_chain(qa, sa, qw, sw, bias, dtype)
    if act == 0:
        return y
    ch = y.step(G.gelu_tanh64, eps=G.gelu_tanh_eps(y.v), turn=G.GELU_TANH_TURN)
    flush = G._K0 * y.lo * (1 + 0.044715 * y.lo * y.lo) > G.TANH_FLUSH_W
    ch.hi = torch.where(flush, torch.clamp_min(ch.hi, 0.0), ch.hi)
    return ch


def fp8_residual_chain(qa, sa, qw, sw, bias, resid, mod, mask, gate_row, B, T, S, dtype):
    N = qw.shape[0]
    y = fp8_linear_chain(qa, sa, qw, sw, bias, dtype)
    y = Chain(*(t.reshape(B, T, S, N) if t.dim() else t for t in (y.lo, y.hi, y.near, y.v, y.eps)), y.dtype)
    if gate_row >= 0:
        y = y.step(lambda yy, g: yy * g, G.mod_row(mod, mask, gate_row, B, T))
    return G._add(y, resid.reshape(B, T, S, N))


def _operands(M, N, K, dtype, seed, a=None, w=None):
    a = _hidden(M, K, dtype=dtype, seed=seed + 1) if a is None else a
    w = _rand(N, K, dtype=dtype, scale=K**-0.5, seed=seed + 2) if w is None else w
    bias = _rand(N, dtype=dtype, scale=0.5, seed=seed + 3)
    qa, sa = kernels.quant_rows_fp8(a)
    qw, sw = kernels.quant_rows_fp8(w)
    return qa, sa, qw, sw, bias


def _twice8(what, fn):
    x, y = fn(), fn()
    assert torch.equal(x.view(torch.int16), y.view(torch.int16)), f"{what}: two launches differ"
    return x


def _assert_fp8_kernel(M, N, K, act=0, residual=False):
    name = kernels.gemm_fp8_kernel_name(M, N, K, act=act, residual=residual)
    assert name == f"gemm_wide_kernel<fp8, {2 if residual else act}>", name


@both
@pytest.mark.parametrize("M,N,K", [(128 * 20 + 1, 1152, 1152), (128 * 20 + 64, 1152, 1152), (128 * 20 + 65, 3456, 1152),
                                   (128 * 20 + 127, 4608, 1152), (128 * 17, 1152, 1168), (1000, 1152, 4608), (7, 8, 16)],
                         ids=["tail1", "tail64", "tail65-N3456", "tail127-N4608", "Ktail1168", "K4608", "tiny"])
@pytest.mark.parametrize("act", [0, 1], ids=["bias", "tanh"])
def test_gemm_fp8_fp64(M, N, K, act, dtype):
    """M tails inside the last 128-row tile (so the second consumer's rows are empty, one row, or full), a K tail inside a
    k-block (K = 1168 = 9 x 128 + 16), OpenSora's output widths 1152 / 3456 / 4608, K = 4608 (mlp.fc2), bias-only and
    tanh-GELU, bf16 and fp16 outputs; two launches give the same bits."""
    _assert_fp8_kernel(M, N, K, act)
    qa, sa, qw, sw, bias = _operands(M, N, K, dtype, seed=M + N + K)
    what = f"gemm_fp8 act={act} M={M} N={N} K={K} {dtype}"
    got = _twice8(what, lambda: kernels.gemm_fp8_bias_act(qa, sa, qw, sw, bias, act))
    assert got.dtype == dtype
    assert _check(what, got, fp8_chain(qa, sa, qw, sw, bias, act, dtype))


@both
def test_gemm_fp8_no_bias(dtype):
    M, N, K = 300, 1152, 1152
    qa, sa, qw, sw, _ = _operands(M, N, K, dtype, seed=3)
    got = kernels.gemm_fp8_bias_act(qa, sa, qw, sw, None, 0, dtype=dtype)
    assert _check(f"gemm_fp8 no bias {dtype}", got, fp8_chain(qa, sa, qw, sw, None, 0, dtype))


@both
@pytest.mark.parametrize("gate_row", [2, 5, -1], ids=["gate2", "gate5", "plain"])
def test_gemm_fp8_residual_epilogue(gate_row, dtype):
    """Gate + per-frame select + residual (every mask pattern) and the plain add, at K = 1152 and 4608: into a separate
    output between NaN guard rows (resid unchanged), and in place, which gives the same bits."""
    failed = []
    for (B, T, S), N, K in (((2, 3, 50), 1152, 1152), ((2, 4, 33), 1152, 4608)):
        M = B * T * S
        _assert_fp8_kernel(M, N, K, residual=True)
        qa, sa, qw, sw, bias = _operands(M, N, K, dtype, seed=N + K)
        resid = _hidden(M, N, dtype=dtype, seed=5)
        mod = _rand(2, B, 6, N, dtype=dtype, scale=0.5, seed=6)
        for mname, mask in _masks(B, T).items():
            if gate_row < 0 and mname != "none":
                continue
            what = f"gemm_fp8 residual {dtype} gate_row={gate_row} M={M} K={K} mask={mname}"
            r0 = resid.clone()
            buf, out = _guarded(M, N, dtype)
            kernels.gemm_fp8_bias_residual(qa, sa, qw, sw, bias, resid, mod, mask, gate_row, B, T, S, out=out)
            _guards_intact(what, buf)
            assert torch.equal(resid, r0), f"{what}: resid changed"
            ibuf, inner = _guarded(M, N, dtype)
            inner.copy_(resid)
            kernels.gemm_fp8_bias_residual(qa, sa, qw, sw, bias, inner, mod, mask, gate_row, B, T, S)
            _guards_intact(what + " in place", ibuf)
            assert torch.equal(inner.view(torch.int16), out.view(torch.int16)), f"{what}: in place differs"
            ch = fp8_residual_chain(qa, sa, qw, sw, bias, resid, mod, mask, gate_row, B, T, S, dtype)
            if not _check(what, out.view(B, T, S, N), ch):
                failed.append(what)
    assert not failed, failed


def test_gemm_fp8_promotion_bound():
    """K = 4608 with products of one sign: a GELU-like activation (>= 0 with a DC offset) against weight rows with a
    positive mean, where the running sum grows with K.  The promoted bound of the module docstring must hold."""
    M, N, K = 512, 1152, 4608
    a = _hidden(M, K, dtype=torch.bfloat16, seed=41).float().abs().to(torch.bfloat16)
    w = (_rand(N, K, dtype=torch.float32, scale=K**-0.5, seed=42) + 0.5 * K**-0.5).to(torch.bfloat16)
    qa, sa, qw, sw, bias = _operands(M, N, K, torch.bfloat16, seed=43, a=a, w=w)
    got = kernels.gemm_fp8_bias_act(qa, sa, qw, sw, bias, 0)
    assert _check("gemm_fp8 one-signed K=4608", got, fp8_chain(qa, sa, qw, sw, bias, 0, torch.bfloat16))


@both
def test_gemm_fp8_30_launches_bit_identical(dtype):
    M, N, K = 36000, 4608, 1152
    qa, sa, qw, sw, bias = _operands(M, N, K, dtype, seed=11)
    ref = kernels.gemm_fp8_bias_act(qa, sa, qw, sw, bias, 1).view(torch.int16).clone()
    out = torch.empty(M, N, dtype=dtype, device=DEV)
    for i in range(30):
        kernels.gemm_fp8_bias_act(qa, sa, qw, sw, bias, 1, out=out)
        assert torch.equal(out.view(torch.int16), ref), f"launch {i} differs"


@both
def test_gemm_fp8_refuses(dtype):
    qa, sa, qw, sw, bias = _operands(64, 1152, 1152, dtype, seed=1)
    with pytest.raises(_lib.VsbError):  # K % 16 != 0
        kernels.gemm_fp8_bias_act(qa[:, :1144].contiguous(), sa, qw[:, :1144].contiguous(), sw, bias)
    with pytest.raises(_lib.VsbError):  # N % 8 != 0
        kernels.gemm_fp8_bias_act(qa, sa, qw[:1148].contiguous(), sw[:1148].contiguous(), bias[:1148].contiguous())
    with pytest.raises(_lib.VsbError):  # erf-GELU has no fp8 instance
        kernels.gemm_fp8_bias_act(qa, sa, qw, sw, bias, 2)


# ---- quantization ----------------------------------------------------------------------------------------------------
def _rows(M, K, dtype, seed):
    """Random rows, rows spanning 2^-20 .. 2^12, all-zero rows, and rows of one outlier among small values."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g)
    x[1::5] *= torch.exp2(torch.randint(-20, 13, (K,), generator=g).float())
    x[2::5] = 0
    x[3::5] *= 1e-3
    x[3::5, 7] = 300.0
    x[4::5] = -x[4::5].abs()
    return x.to(dtype).to(DEV)


def _bits_equal(what, got, want):
    g, w = got.view(torch.uint8), want.view(torch.uint8)
    bad = int((g != w).sum())
    assert bad == 0, f"{what}: {bad} of {g.numel()} codes differ"


@both
@pytest.mark.parametrize("K", [8, 1152, 1160, 4608])
def test_quant_rows_fp8_bit_exact(K, dtype):
    x = _rows(257, K, dtype, seed=K)
    q, s = kernels.quant_rows_fp8(x)
    rq, rs = fp8_rule.quant_rows(x.cpu())
    _bits_equal(f"quant K={K} {dtype}", q.cpu(), rq)
    assert torch.equal(s.cpu(), rs)
    assert bool((s.cpu()[2::5] == 1).all()) and bool((q.cpu().view(torch.uint8)[2::5] == 0).all())


@both
@pytest.mark.parametrize("C", [1152, 2304, 3072])
def test_ln_modulate_fp8_is_ln_modulate_then_quant(C, dtype):
    """Fused == unfused bit for bit, and both == the rule on the 16-bit rows: every x_mask pattern, and zero rows (a
    constant input row normalises to 0; sample 1's shift row is zero there)."""
    B, T, S = 2, 4, 37
    x = _hidden(B, T * S, C, dtype=dtype, seed=C)
    x[1, :S] = 0.25  # constant rows of sample 1, frame 0
    mod = _rand(2, B, 6, C, dtype=dtype, scale=0.5, seed=C + 1)
    mod[:, 1, 0] = 0  # shift row of sample 1: zero output rows
    for mname, mask in _masks(B, T).items():
        for sh, sc in ((0, 1), (3, 4)):
            what = f"ln_modulate_fp8 C={C} {dtype} mask={mname} rows={sh},{sc}"
            y = kernels.ln_modulate(x, mod, mask, sh, sc, B, T, S)
            q, s = kernels.ln_modulate_fp8(x, mod, mask, sh, sc, B, T, S)
            uq, us = kernels.quant_rows_fp8(y)
            _bits_equal(what, q, uq)
            assert torch.equal(s, us), what
            rq, rs = fp8_rule.quant_rows(y.cpu())
            _bits_equal(what + " vs rule", q.cpu(), rq)
            assert torch.equal(s.cpu(), rs), what
            if sh == 0 and mname == "none":
                assert bool((s[1, :S] == 1).all()) and bool((q[1, :S].view(torch.uint8) == 0).all()), what
