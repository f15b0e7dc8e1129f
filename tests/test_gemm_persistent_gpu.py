"""The persistent ping-pong GEMM (GELU epilogues at short K, every gate + residual epilogue): tile counts against the grid (min(tiles, SMs) CTAs, two consumers per CTA taking
alternate 128 x 128 tiles) and the fused residual epilogue, whose resid block arrives by TMA in the staging tile, over
many tiles per CTA, in bf16 and in the IEEE fp16 twin.  Same tolerances as test_kernels_gpu.py."""
import pytest
import torch

from oracle import stdit3_oracle as O, synth
from tests.test_kernels_gpu import _dev, _gemm_check, _mask_u8, _ulp_report

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


@pytest.mark.parametrize("case", ["tiles_not_multiple", "fewer_tiles_than_sms", "odd_tiles_per_cta", "even_tiles_plus_one"])
@pytest.mark.parametrize("dt", [BF, F16])
def test_gemm_tile_counts(case, dt):
    """350 tiles (not a multiple of the grid), 27 tiles (fewer CTAs than SMs, one tile each: the second consumer idles),
    3 tiles per CTA (the last falls to the first consumer), 2 per CTA + a remainder (the last falls to either).  All with
    the tanh-GELU epilogue at K <= 1536, which runs on the persistent kernel (a bias-only GEMM does not)."""
    sms = _sms()
    M, N, K_, act = {
        "tiles_not_multiple": (128 * 50 - 37, 128 * 7, 576, 1),
        "fewer_tiles_than_sms": (300, 1152, 1152, 1),
        "odd_tiles_per_cta": (128 * 3 * sms // 9, 1152, 320, 1),
        "even_tiles_plus_one": (128 * (2 * sms + 1), 128, 192, 1),
    }[case]
    _gemm_check(f"pp.{case}", M, N, K_, act, BF=dt)


@pytest.mark.parametrize("dt", [BF, F16])
@pytest.mark.parametrize("B,T,S,N,K_,gate_row,separate_out", [
    (2, 8, 701, 1152, 1152, 2, False),   # attn.proj: ~6 tiles per CTA, M tail, gate + frame select, in place
    (2, 4, 333, 1152, 4608, 5, False),   # mlp.fc2: long K, gate + frame select, in place
    (2, 8, 701, 1152, 1152, -1, False),  # cross_attn.proj: plain residual add, in place
    (1, 3, 500, 520, 256, -1, True),     # N % 128 != 0 (a 64-column chunk outside N), out != resid
])
def test_gemm_fused_residual_many_tiles(B, T, S, N, K_, gate_row, separate_out, dt):
    from videosys_b200 import kernels as K

    dev = _dev()
    M = B * T * S
    tag = f"ppr{M}x{N}x{K_}"
    a = synth.normalish(f"{tag}.a", (M, K_)).to(dt)
    w = synth.normalish(f"{tag}.w", (N, K_), std=0.05).to(dt)
    bias = (0.1 * synth.uniform(f"{tag}.b", (N,))).to(dt)
    x = synth.normalish(f"{tag}.x", (B, T * S, N)).to(dt)
    y = torch.nn.functional.linear(a, w, bias).reshape(B, T * S, N)
    xg = x.to(dev).clone()
    out = torch.empty_like(xg) if separate_out else None
    if gate_row >= 0:
        table = synth.normalish(f"{tag}.tab", (6, N), std=0.3).to(dt)
        t = synth.normalish(f"{tag}.t", (B, 6 * N), std=0.5).to(dt)
        t0 = synth.normalish(f"{tag}.t0", (B, 6 * N), std=0.5).to(dt)
        x_mask = torch.ones(B, T, dtype=torch.bool)
        x_mask[0, 1] = False
        x_mask[B - 1, T - 1] = False
        mods = table[None] + t.reshape(B, 6, N)
        mods0 = table[None] + t0.reshape(B, 6, N)
        branch = O.frame_select(x_mask, mods[:, gate_row:gate_row + 1] * y, mods0[:, gate_row:gate_row + 1] * y, T, S)
        want = x + branch
        mod = torch.stack([mods, mods0]).contiguous().to(dev)  # [2, B, 6, N]: t rows, then t0 rows
        got = K.gemm_bias_residual(a.to(dev), w.to(dev), bias.to(dev), xg, mod, _mask_u8(x_mask, dev), gate_row, B, T, S, out=out)
    else:
        branch = y
        want = x + y
        got = K.gemm_bias_residual(a.to(dev), w.to(dev), bias.to(dev), xg, out=out)
    if separate_out:
        assert torch.equal(xg.cpu(), x), "resid is read only when out is separate"
    else:
        assert got.data_ptr() == xg.data_ptr(), "the fused kernel updates x in place"
    # a one-ulp accumulation-order flip of the branch survives the residual add: measure in ulps of max(|sum|, |branch|)
    _ulp_report(f"gemm+residual {dt} M={M} N={N} K={K_} gate_row={gate_row}", got.reshape(B, T * S, N), want, min_equal=0.98,
                max_ulps=3.0, row_floor=0.25, bits=8 if dt == BF else 11, mag_floor=branch)
