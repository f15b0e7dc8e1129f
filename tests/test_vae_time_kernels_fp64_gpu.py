"""The SVD temporal decoder's kernels on the H100, every output element against float64 with the rule of
tests/vae_fp64.py, in bf16 and fp16: vae_conv_time (a (3, 1, 1) convolution over zero-padded frames, with and without
the residual + AlphaBlender epilogue) on 8 x 16 tile seams and H / W that are not multiples of the tile, written into
NaN-fenced output frames; and vae_time_conv_rgb (time_conv_out on RGB)."""
import pytest
import torch
import torch.nn.functional as F

from tests import vae_fp64 as V
from videosys_b200 import kernels

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


def _time_conv64(x, w):
    """float64 (kt, 1, 1) convolution of x [B, kt-1+T, H, W, Cin] and the same of the squares (for eps)."""
    xi, wd = x.permute(0, 4, 1, 2, 3).double(), w.double()
    return F.conv3d(xi, wd).permute(0, 2, 3, 4, 1), F.conv3d(xi * xi, wd * wd).permute(0, 2, 3, 4, 1)


def conv_time_chain(x, w, bias, resid=None, mix=None):
    """r(r(conv) + bias), then r(. + resid), or with mix = (a, b): xt = r(resid + v), r(r(a * resid) + r(b * xt))."""
    dt = x.dtype
    conv, sq = _time_conv64(x, w)
    K = w[0].numel()
    b = bias.double()
    ch = V.Chain.start(conv, V.sum_eps(sq, K) + (K / 16) * V.U32 * conv.abs(), dt)
    ch = ch.step(lambda c, bb: c + bb, b, eps=V.U32 * (conv.abs() + b.abs()))
    if resid is None:
        return ch
    r = resid.double()
    ch = ch.step(lambda y, rr: y + rr, r, eps=V.U32 * (ch.v.abs() + r.abs()))
    if mix is None:
        return ch
    a, bm = mix
    assert bm > 0
    pa = V.Chain.start(a * r, 0.0, dt)  # a product of two 16-bit values is exact in fp32
    pb = ch.step(lambda t: bm * t)
    return pb.step(lambda q, p: q + p, pa, eps=V.U32 * (pb.v.abs() + pa.v.abs()))


def _regions(B, T, H, W):
    y = torch.arange(H, device=DEV).view(H, 1)
    x = torch.arange(W, device=DEV).view(1, W)
    border = (y == 0) | (y == H - 1) | (x == 0) | (x == W - 1)
    seam = (((x % 16 == 0) | (x % 16 == 15)) | ((y % 8 == 0) | (y % 8 == 7))) & ~border
    return {k: m.expand(B, T, H, W) for k, m in (("border", border), ("seam", seam), ("interior", ~border & ~seam))}


def _mix(m, dtype):
    """The AlphaBlender's (a, b) of mix_factor m as the model computes them in the parameter dtype."""
    a = 1.0 - torch.sigmoid(torch.tensor([m], dtype=dtype, device=DEV))
    return float(a), float(1.0 - a)


CASES = {  # name: (B, T, H, W, C)
    "128_t14_40x50": (1, 14, 40, 50, 128),
    "128_t1_b2_13x21": (2, 1, 13, 21, 128),
    "256_t2_17x33": (1, 2, 17, 33, 256),
    "256_t14_b2_9x7": (2, 14, 9, 7, 256),
    "512_t14_8x16": (1, 14, 8, 16, 512),
    "512_t2_b2_5x7": (2, 2, 5, 7, 512),
    "512_t1_1x1": (1, 1, 1, 1, 512),
}


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("mode", ["plain", "resid", "mix"])
@pytest.mark.parametrize("name", list(CASES))
def test_vae_conv_time_fp64(name, mode, dtype):
    B, T, H, W, C = CASES[name]
    x = torch.zeros(B, T + 2, H, W, C, dtype=dtype, device=DEV)  # padding (1, 0, 0): frames 0 and T+1 stay zero
    x[:, 1:T + 1] = _act(B, T, H, W, C, dtype=dtype, seed=1)
    w = _rand(C, C, 3, 1, 1, dtype=dtype, scale=(C * 3) ** -0.5, seed=2)
    bias = _rand(C, dtype=dtype, scale=0.1, seed=3)
    xs = _act(B, T, H, W, C, dtype=dtype, seed=4, offset=-0.2) if mode != "plain" else None
    mix = _mix(0.7 if name.startswith("128") else -1.3, dtype) if mode == "mix" else None
    got = kernels.vae_conv_time(x, kernels.pack_conv_weight(w), bias, C, 3, resid=xs, mix=mix)
    assert got.shape == (B, T, H, W, C)
    ch = conv_time_chain(x, w, bias, xs, mix)
    failed = [where for where, m in _regions(B, T, H, W).items()
              if bool(m.any()) and not V.check(f"conv_time {name} {mode} {dtype} {where}", got, ch, mask=m)[0]]
    assert not failed, f"outside the legal set in {failed}"


def _on_nan_memory(shape, dtype, fn):
    """fn() with the caching allocator's next block of `shape` filled with NaN first: an output element the kernel does
    not write stays NaN."""
    torch.cuda.synchronize()
    torch.full(shape, float("nan"), dtype=dtype, device=DEV)
    return fn()


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_vae_conv_time_writes_every_output_and_reads_no_padding_garbage(dtype):
    """Every output element is written (NaN-filled output memory), and the zero frames around the input are what the
    kernel reads at the ends of the clip (NaN frames beyond them are not read)."""
    B, T, H, W, C = 2, 3, 9, 17, 128
    x = torch.full((B, T + 4, H, W, C), float("nan"), dtype=dtype, device=DEV)  # NaN fences around the padded clip
    x[:, 1] = 0
    x[:, T + 2] = 0
    x[:, 2:T + 2] = _act(B, T, H, W, C, dtype=dtype, seed=5)
    xin = x[:, 1:T + 3].contiguous()
    w = _rand(C, C, 3, 1, 1, dtype=dtype, scale=(C * 3) ** -0.5, seed=6)
    bias = _rand(C, dtype=dtype, scale=0.1, seed=7)
    xs = _act(B, T, H, W, C, dtype=dtype, seed=8)
    mix = _mix(0.0, dtype)
    out = _on_nan_memory((B, T, H, W, C), dtype, lambda: kernels.vae_conv_time(xin, kernels.pack_conv_weight(w), bias, C, 3,
                                                                              resid=xs, mix=mix))
    assert not bool(torch.isnan(out.float()).any())
    V.assert_legal(f"conv_time mix {dtype}", out, conv_time_chain(xin, w, bias, xs, mix))


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_vae_conv_time_mix_epilogue_equals_unfused_passes(dtype):
    """The fused epilogue is bit for bit the residual epilogue followed by vae_mix (a * xs + b * xt, each op rounded)."""
    B, T, H, W, C = 1, 14, 24, 40, 256
    x = torch.zeros(B, T + 2, H, W, C, dtype=dtype, device=DEV)
    x[:, 1:T + 1] = _act(B, T, H, W, C, dtype=dtype, seed=12)
    wp = kernels.pack_conv_weight(_rand(C, C, 3, 1, 1, dtype=dtype, scale=(C * 3) ** -0.5, seed=13))
    bias = _rand(C, dtype=dtype, scale=0.1, seed=14)
    xs = _act(B, T, H, W, C, dtype=dtype, seed=15)
    a, b = _mix(0.4, dtype)
    fused = kernels.vae_conv_time(x, wp, bias, C, 3, resid=xs, mix=(a, b))
    V.assert_bit_exact(f"conv_time mix fused vs unfused {dtype}", fused,
                       kernels.vae_mix(xs, kernels.vae_conv_time(x, wp, bias, C, 3, resid=xs), a, b))


RGB_CASES = {"t14_512x512": (1, 14, 512, 512), "t1_b2_13x21": (2, 1, 13, 21), "t2_40x50": (1, 2, 40, 50), "t16_b2_7x9": (2, 16, 7, 9)}


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", list(RGB_CASES))
def test_vae_time_conv_rgb_fp64(name, dtype):
    B, T, H, W = RGB_CASES[name]
    x = _rand(B, T, H, W, 3, dtype=dtype, seed=9)
    w = _rand(3, 3, 3, 1, 1, dtype=dtype, scale=0.3, seed=10)
    bias = _rand(3, dtype=dtype, scale=0.1, seed=11)
    got = _on_nan_memory(x.shape, dtype, lambda: kernels.vae_time_conv_rgb(x, w, bias))
    assert not bool(torch.isnan(got.float()).any())
    xp = F.pad(x, (0, 0, 0, 0, 0, 0, 1, 1))  # zero frames at both ends
    V.assert_legal(f"time_conv_rgb {name} {dtype}", got, conv_time_chain(xp, w, bias))
