"""OpenSora v1.2 VAE encoder on the H100: the strided convolution (vae_conv_down) and the Cout = 8 epilogue element by
element against float64 (the rule of tests/vae_fp64.py) with NaN sentinels around the output, 30 launches bit-identical;
the whole encoder's posterior means against the reference's fp32 outputs within 1.25x of the eager 16-bit chain's own
error, and a seeded encode against the eager 16-bit chain drawing the same noise."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle.gen_golden_opensora_vae import weights
from oracle.gen_golden_opensora_vae_encode import CASES, SEED, sample_index, videos
from tests import kernels_emul_vae_down as ED
from tests import vae_fp64 as V
from videosys_b200 import _lib, kernels
from videosys_b200.models.autoencoders import OpenSoraVAEEncoder

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _act(*shape, dtype, seed, offset=0.3):
    """Activations, channels last: every third channel post-SiLU, a DC offset, four channels x 20."""
    z = torch.randn(*shape, generator=_gen(seed))
    z[..., ::3] = F.silu(2 * z[..., ::3])
    z = z + offset
    z[..., :4] *= 20
    return z.to(dtype).to(DEV)


def _rand(*shape, dtype, scale=1.0, seed=0):
    return (scale * torch.randn(*shape, generator=_gen(seed))).to(dtype).to(DEV)


def down_chain(x, w, bias, kt):
    """vae_conv_down of x [B, Tin, Hin, Win, Cin] with w [Cout, Cin, kt, 3, 3]: the float64 strided convolution (kt = 1:
    zero pad right / bottom by 1, stride (1, 2, 2); kt = 3: one zero frame in front, zero pad 1 spatially, stride
    (2, 1, 1)), then r(r(conv) + b)."""
    xi = x.permute(0, 4, 1, 2, 3).double()
    xi, stride = (F.pad(xi, (0, 1, 0, 1)), (1, 2, 2)) if kt == 1 else (F.pad(xi, (1, 1, 1, 1, 1, 0)), (2, 1, 1))
    wd = w.double()
    conv = F.conv3d(xi, wd, stride=stride).permute(0, 2, 3, 4, 1)
    sq = F.conv3d(xi * xi, wd * wd, stride=stride).permute(0, 2, 3, 4, 1)
    K = w[0].numel()
    eps_sum = V.sum_eps(sq, K) + (K / 16) * V.U32 * conv.abs()  # as tests/vae_fp64.conv_chain
    b = bias.double()
    return V.Chain.start(conv, eps_sum, x.dtype).step(lambda c, bb: c + bb, b, eps=V.U32 * (conv.abs() + b.abs()))


# name: (B, Tin, Hin, Win, Cin, Cout, kt)
DOWN_CASES = {
    "hw_16to64_13x21": (2, 1, 13, 21, 16, 64, 1),       # odd H and W: the far-side pad is read
    "hw_64to128_30x46": (1, 2, 30, 46, 64, 128, 1),     # even H, W: the pad is never read
    "hw_128_90x160": (1, 1, 90, 160, 128, 128, 1),      # partial edge tiles (45 x 80 out)
    "hw_512_45x80": (2, 1, 45, 80, 512, 512, 1),
    "hw_256to8_17x35": (1, 1, 17, 35, 256, 8, 1),
    "t_256_8x13x21": (1, 8, 13, 21, 256, 256, 3),       # the zero frame in front is frame -1's fill: 8 frames -> 4
    "t_64to128_4x30x45_b2": (2, 4, 30, 45, 64, 128, 3),
    "t_16to64_2x8x16": (1, 2, 8, 16, 16, 64, 3),
    "t_512to8_7x5x7": (1, 7, 5, 7, 512, 8, 3),          # odd: the last frame is read only as frame 2t + 1 of t = 2
}


def _launch_into(x, wp, b, cout, kt, out):
    """vsb_vae_conv_down straight into `out` (a frame window of a larger NaN-filled buffer)."""
    B, Tin, Hin, Win, Cin = x.shape
    lib, st = kernels._prep(x, wp, b)
    _lib.check(kernels._fn(lib, "vsb_vae_conv_down", x)(x.data_ptr(), wp.data_ptr(), b.data_ptr(), out.data_ptr(), B, Tin,
                                                         Hin, Win, Cin, cout, kt, 2 if kt == 3 else 1, 1 if kt == 3 else 2,
                                                         1, st), "vae_conv_down")


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("name", list(DOWN_CASES))
def test_vae_conv_down_fp64(name, dtype):
    B, Tin, Hin, Win, Cin, Cout, kt = DOWN_CASES[name]
    x = _act(B, Tin, Hin, Win, Cin, dtype=dtype, seed=1)
    w = _rand(Cout, Cin, kt, 3, 3, dtype=dtype, scale=(Cin * kt * 9) ** -0.5, seed=2)
    b = _rand(Cout, dtype=dtype, scale=0.1, seed=3)
    wp = kernels.pack_conv_weight(w)
    got = kernels.vae_conv_down(x, wp, b, Cout, kt)
    T, H, W = ((Tin, (Hin - 2) // 2 + 1, (Win - 2) // 2 + 1) if kt == 1 else ((Tin - 2) // 2 + 1, Hin, Win))
    assert got.shape == (B, T, H, W, Cout)
    V.assert_legal(f"conv_down {name} {dtype}", got, down_chain(x, w, b, kt))
    flat = torch.full(((B * T + 2) * H * W * Cout,), float("nan"), dtype=dtype, device=DEV)
    _launch_into(x, wp, b, Cout, kt, flat[H * W * Cout:])
    assert bool(torch.isnan(flat[:H * W * Cout].float()).all()) and bool(torch.isnan(flat[-H * W * Cout:].float()).all()), \
        "wrote outside the output"
    assert torch.equal(flat[H * W * Cout:-H * W * Cout].view(got.shape), got)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_vae_conv_down_repeat_bit_identical(dtype):
    x = _act(1, 1, 90, 160, 128, dtype=dtype, seed=5)
    w = _rand(128, 128, 1, 3, 3, dtype=dtype, scale=(128 * 9) ** -0.5, seed=6)
    b = _rand(128, dtype=dtype, scale=0.1, seed=7)
    wp = kernels.pack_conv_weight(w)
    first = kernels.vae_conv_down(x, wp, b, 128, 1)
    for _ in range(29):
        assert torch.equal(kernels.vae_conv_down(x, wp, b, 128, 1), first)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("H,W,Cin", [(90, 160, 512), (13, 21, 128)])
def test_vae_conv3d_cout8_fp64(H, W, Cin, dtype):
    """The image encoder's conv_out: 3x3, Cout = 8, per image (kt = 1)."""
    x = _act(2, 1, H, W, Cin, dtype=dtype, seed=8)
    w = _rand(8, Cin, 1, 3, 3, dtype=dtype, scale=(Cin * 9) ** -0.5, seed=9)
    b = _rand(8, dtype=dtype, scale=0.1, seed=10)
    got = kernels.vae_conv3d(x, kernels.pack_conv_weight(w), b, 8, 1)
    V.assert_legal(f"conv3d Cout=8 {H}x{W} {dtype}", got, V.conv_chain(x, w, b))


# ---- the whole encoder ----
@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", "opensora_vae_encode.pt"))


def _enc(name, dtype=torch.bfloat16):
    enc = OpenSoraVAEEncoder(spatial_block_out_channels=CASES[name][0])
    enc.load_state_dict(weights(enc.state_dict(), name))
    return enc.to(dtype).to(DEV).eval()


def _eager(monkeypatch, fn):
    with monkeypatch.context() as m:
        for n, f in ED.stand_ins().items():
            m.setattr(kernels, n, f)
        return fn()


def _zero_noise(m):
    m.setattr(torch, "randn", lambda *s, **kw: torch.zeros(*s, **{k: v for k, v in kw.items() if k != "generator"}))


@pytest.mark.parametrize("name", list(CASES))
def test_opensora_vae_encode_golden_within_eager16_error(monkeypatch, gold, name):
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    enc = _enc(name)
    x = videos(name).to(DEV)
    with monkeypatch.context() as m:
        _zero_noise(m)
        n0 = kernels.launch_count()
        ours = enc.encode(x)
        assert kernels.launch_count() - n0 > 50
        assert torch.equal(ours, enc.encode(x)), "two encodes differ"
        eager = _eager(monkeypatch, lambda: enc.encode(x))
    assert list(ours.shape) == gold[f"{name}.shape"]
    want = gold[f"{name}.mode"].double()
    idx = sample_index(ours.numel(), name).to(DEV) if ours.numel() > want.numel() else torch.arange(ours.numel(), device=DEV)
    e_ours = float((ours.flatten()[idx].double().cpu() - want).norm())
    e_eager = float((eager.flatten()[idx].double().cpu() - want).norm())
    print(f"[encode {name}] |ours - ref| = {e_ours:.4g}, |eager16 - ref| = {e_eager:.4g}, ratio {e_ours / e_eager:.3f}")
    assert e_ours <= 1.25 * e_eager


def test_opensora_vae_encode_seeded_draws_match_eager(monkeypatch):
    """With noise, under one seed: the native encode and the eager 16-bit chain draw the same CUDA and CPU noise."""
    enc = _enc("remainder")
    x = videos("remainder").to(DEV)
    torch.manual_seed(SEED)
    ours = enc.encode(x)
    torch.manual_seed(SEED)
    eager = _eager(monkeypatch, lambda: enc.encode(x))
    rel = float((ours.double() - eager.double()).norm() / eager.double().norm())
    print(f"[encode seeded] rel L2 native vs eager16 = {rel:.3e}")
    assert rel < 5e-2
