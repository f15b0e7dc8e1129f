"""The 256 x 128 persistent GEMM (gemm_wide_kernel in csrc/gemm_wgmma.cu) element by element against float64, through the
public entries at shapes the dispatch sends to it (2048 tiles or more; the residual epilogue only at K >= 4608): M
tails inside the last 256-row panel (a last panel of 1, 127, 128, 129 or 255 rows, so the second consumer's half is
empty, partly filled or full), a K tail, tile counts that are not a multiple of the grid (15 to 16 tiles per CTA),
tanh- and erf-GELU, the gate + per-frame select + residual
with mixed frame flags and the plain residual add, in place and into a separate output framed by NaN guard rows,
bf16 and fp16, and 30 launches bit for bit.  The reference chains and the acceptance rule are those of
tests/test_gemm_attn_kernels_fp64_gpu.py."""
import pytest
import torch

from tests import gemm_attn_fp64 as G
from tests.test_dit_kernels_fp64_gpu import _masks
from tests.test_gemm_attn_kernels_fp64_gpu import (DEV, DTYPES, EPI, IDS, _check, _gemm_inputs, _guarded, _guards_intact,
                                                   _hidden, _rand, _twice)
from videosys_b200 import kernels

pytestmark = pytest.mark.gpu
both = pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
N0 = 1152  # OpenSora's hidden width: 9 column tiles


MIN_TILES = 2048  # kWideMinTiles


def _panels(n_tiles):
    """256-row panels that make at least MIN_TILES tiles of n_tiles column tiles."""
    return -(-MIN_TILES // n_tiles)


def _assert_wide(M, N, K, act=0, residual=False):
    name = kernels.gemm_kernel_name(M, N, K, act=act, residual=residual)
    assert name.startswith("gemm_wide_kernel"), f"M={M} N={N} K={K} act={act} residual={residual} runs {name}"


def _run(what, M, N, K, act, dtype, bias=True):
    _assert_wide(M, N, K, EPI[act])
    a, w, b = _gemm_inputs(M, N, K, dtype, seed=M + K)
    b = b if bias else None
    got = _twice(what, lambda: kernels.gemm_bias_act(a, w, b, EPI[act]))
    return _check(what, got, G.gemm_chain(a, w, b, act))


@both
@pytest.mark.parametrize("tail", [1, 127, 128, 129, 255])
def test_gemm_wide_m_tails(tail, dtype):
    """Bias only, M % 256 = tail: the last panel's second half is empty (1, 127, 128) or partly inside M; K = 136 ends in
    a partial k-block.  2052 tiles: 15 or 16 per CTA on 132 SMs, not a multiple of the grid."""
    M = 256 * (_panels(N0 // 128) - 1) + tail
    assert _run(f"wide M={M} tail={tail} {dtype}", M, N0, 136, 0, dtype, bias=tail != 128)


@both
@pytest.mark.parametrize("act,K", [(1, 1152), (1, 2304), (3, 1152), (3, 2304)], ids=["tanh1152", "tanh2304", "erf1152",
                                                                                 "erf2304"])
def test_gemm_wide_gelu(act, K, dtype):
    """The tanh- and erf-GELU epilogues (applied by the epilogue warps to the staged bf16(acc + bias)) at K = 1152, where
    the K loop that hides them is shortest, and at K = 2304; 36 column tiles."""
    M = 256 * _panels(36) - 3
    assert _run(f"wide act={act} M={M} K={K} {dtype}", M, 4608, K, act, dtype)


@both
@pytest.mark.parametrize("gate_row", [5, -1], ids=["gate5", "plain"])
def test_gemm_wide_residual_epilogue(gate_row, dtype):
    """mlp.fc2's epilogue at K = 4608: gate row 5 with the t and t0 rows mixed inside tiles (the first frame of the first
    sample and the last of the last take t0; S = 4851 is not a multiple of 256), and the plain add.  M % 256 = 100, so
    the last panel's second half gets no resid load.  Into a separate output between NaN guard rows (resid unchanged),
    and in place."""
    B, T, S, N, K = 2, 6, 4851, N0, 4608
    M = B * T * S
    _assert_wide(M, N, K, residual=True)
    a, w, bias = _gemm_inputs(M, N, K, dtype, seed=N + K)
    resid = _hidden(M, N, dtype=dtype, seed=5)
    mod = _rand(2, B, 6, N, dtype=dtype, scale=0.5, seed=6)
    mask = _masks(B, T)["first/last off"] if gate_row >= 0 else None
    what = f"wide residual {dtype} gate_row={gate_row} M={M} K={K}"
    r0 = resid.clone()
    buf, out = _guarded(M, N, dtype)
    kernels.gemm_bias_residual(a, w, bias, resid, mod, mask, gate_row, B, T, S, out=out)
    _guards_intact(what, buf)
    assert torch.equal(resid, r0), f"{what}: resid changed"
    ibuf, inner = _guarded(M, N, dtype)
    inner.copy_(resid)
    kernels.gemm_bias_residual(a, w, bias, inner, mod, mask, gate_row, B, T, S)
    _guards_intact(what + " in place", ibuf)
    assert torch.equal(inner, out), f"{what}: in place differs"
    assert _check(what, out.view(B, T, S, N), G.gemm_residual_chain(a, w, bias, resid, mod, mask, gate_row, B, T, S))


@both
def test_gemm_wide_30_launches_bit_identical(dtype):
    """30 launches of a tanh-GELU GEMM at 36 000 x 4608 x 1536 (5076 tiles) give the same bits."""
    M, N, K = 36000, 4608, 1536
    _assert_wide(M, N, K, act=1)
    a, w, bias = _gemm_inputs(M, N, K, dtype, seed=11)
    ref = kernels.gemm_bias_act(a, w, bias, 1).view(torch.int16).clone()
    out = torch.empty(M, N, dtype=dtype, device=DEV)
    for i in range(30):
        kernels.gemm_bias_act(a, w, bias, 1, out=out)
        assert torch.equal(out.view(torch.int16), ref), f"launch {i} differs"
