"""The float64 reference chains of tests/gemm_attn_fp64.py on small CPU tensors, in bf16 and fp16: every chain accepts an
fp32 emulation of its kernel's arithmetic (the GEMM with truncating k16 accumulation, the tiled online softmax with fp32 l
and 16-bit P in the tile frame at both tile sizes, the eager attn_short chain), and rejects a seeded mutation of it, one
per class of kernel bug.  This is the evidence that tests/test_gemm_attn_kernels_fp64_gpu.py is neither blind nor
over-strict, without a GPU."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import gemm_attn_fp64 as G
from tests import kernels_emul as E
from tests import vae_fp64 as V

DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]
both = pytest.mark.parametrize("dtype", DTYPES, ids=IDS)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rand(*shape, dtype, scale=1.0, offset=0.0, seed=0):
    return (offset + scale * torch.randn(*shape, generator=_gen(seed))).to(dtype)


def _hidden(*shape, dtype, seed, offset=0.3):
    """DiT-like hidden states: a DC offset and four channels x 20."""
    z = offset + torch.randn(*shape, generator=_gen(seed))
    z[..., 3:7] *= 20
    return z.to(dtype)


def _accepts(what, got, chain):
    st = V.assert_legal(what, got, chain)
    G.legal_report(chain)
    return st


def _rejects(what, got, chain):
    ok, st = V.check(what, got, chain)
    assert not ok and st["bad"] > 0, f"{what} was accepted"


# ---------------------------------------------------------------------------------------------------------------------
# GEMM: fp32 emulation with truncating k16 accumulation
# ---------------------------------------------------------------------------------------------------------------------
def trunc32(x):
    """float64 x truncated towards zero to fp32 precision (subnormal spacing below 2^-126)."""
    _, e = torch.frexp(x)
    e = torch.clamp(e.long() - 24, min=-149)
    u = ((e + 1023) << 52).view(torch.float64)
    return torch.trunc(x / u) * u


def _acc(a, w, drop_kblock=False, drop_last_k=False):
    ad, wd = a.double(), w.double()
    K = a.shape[1]
    if drop_kblock:
        ad = ad.clone()
        ad[:, 64:128] = 0
    if drop_last_k:
        ad = ad.clone()
        ad[:, K - 1] = 0
    acc = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float64)
    for k0 in range(0, K, 16):
        acc = trunc32(acc + ad[:, k0:k0 + 16] @ wd[:, k0:k0 + 16].T)
    return acc.float()


def _gelu_tanh_kernel(x):
    """gelu_tanh_f in fp32 torch ops: x / (1 + 2^w), w = x (x^2 kC1 + kC0)."""
    k0 = torch.tensor(-2.0 * 0.7978845608028654, dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32)
    k1 = k0 * torch.tensor(0.044715, dtype=torch.float32)
    w = x * (x * x * k1 + k0)
    return x / (1 + torch.exp2(w))


def _gelu_erf_kernel(x):
    """gelu_erf_f in fp32 torch ops, erff correctly rounded (inside its 2-ulp bound; torch's CPU erf is not)."""
    z = x * torch.tensor(0.70710678118654752440, dtype=torch.float32)
    return x * 0.5 * (1 + torch.erf(z.double()).float())


def _gemm_eager(a, w, bias, act, bug=None):
    dt = a.dtype
    acc = _acc(a, w, drop_kblock=bug == "drop_kblock", drop_last_k=bug == "drop_last_k")
    b = torch.zeros(w.shape[0]) if bias is None else bias.float()
    if bug == "bias_after_round":
        y = (acc.to(dt).float() + b).to(dt)
    elif bug == "truncate" and act == 0:
        return V.round16((acc + b).double(), dt, mode="zero").to(dt)
    else:
        y = (acc + b).to(dt)
    x = (acc + b) if bug == "gelu_unrounded" else y.float()
    if act == 1:
        return _gelu_tanh_kernel(x).to(dt)
    if act == 3:
        return (_gelu_tanh_kernel(x) if bug == "tanh_for_erf" else _gelu_erf_kernel(x)).to(dt)
    return y


def _gemm_case(dtype, M=24, N=40, K=256, cancel=False, seed=0):
    a = _hidden(M, K, dtype=dtype, seed=seed + 1, offset=8.0 if cancel else 0.3)
    w = torch.randn(N, K, generator=_gen(seed + 2)) * 0.05
    if cancel:
        w = w - w.mean(1, keepdim=True)  # zero-mean rows against a DC-offset A: partial sums far above the result
        w[:, 3:7] = 0  # (the massive channels would otherwise dominate the result)
    w = w.to(dtype)
    bias = _rand(N, dtype=dtype, scale=0.5, seed=seed + 3)
    return a, w, bias


@both
@pytest.mark.parametrize("act", [0, 1, 3], ids=["none", "tanh", "erf"])
@pytest.mark.parametrize("shape", [(24, 40, 256), (1, 8, 8), (7, 16, 24), (5, 24, 72)], ids=lambda s: "x".join(map(str, s)))
def test_gemm_chain_accepts_emulation(shape, act, dtype):
    M, N, K = shape
    a, w, bias = _gemm_case(dtype, M, N, K)
    for bb in (bias, None):
        _accepts(f"gemm act={act} {shape} bias={bb is not None}", _gemm_eager(a, w, bb, act), G.gemm_chain(a, w, bb, act))


@both
@pytest.mark.parametrize("act", [0, 1, 3], ids=["none", "tanh", "erf"])
def test_gemm_chain_accepts_cancellation(act, dtype):
    """A DC-offset A against zero-mean W rows: the truncation of large partial sums is inside the rule."""
    a, w, bias = _gemm_case(dtype, 16, 32, 1024, cancel=True)
    acc, _ = G.acc_core(a, w)
    partial = torch.cumsum((a.double().view(16, 1, 64, 16) * w.double().view(1, 32, 64, 16)).sum(3), 2).abs().amax(2)
    assert float((partial / acc.abs()).median()) > 2  # the case does what it says: partial sums above the result
    _accepts(f"gemm cancellation act={act}", _gemm_eager(a, w, bias, act), G.gemm_chain(a, w, bias, act))


@both
@pytest.mark.parametrize("act", [1, 3], ids=["tanh", "erf"])
def test_gelu_chain_accepts_every_16_bit_value(act, dtype):
    """The epilogue over its whole input range: out[n] = act(w[n, 0]) for every finite 16-bit value."""
    allv = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype)
    x = allv[torch.isfinite(allv.float())]
    x = torch.cat([x, torch.zeros((-x.numel()) % 8, dtype=dtype)])
    a = torch.zeros(1, 8, dtype=dtype)
    a[0, 0] = 1
    w = torch.zeros(x.numel(), 8, dtype=dtype)
    w[:, 0] = x
    ch = G.gemm_chain(a, w, None, act)
    ref = (_gelu_tanh_kernel(x.float()) if act == 1 else _gelu_erf_kernel(x.float())).to(dtype)
    _accepts(f"gelu act={act} all values", ref.view(1, -1), ch)


@both
@pytest.mark.parametrize("bug,act", [("drop_kblock", 0), ("drop_last_k", 0), ("bias_after_round", 0), ("gelu_unrounded", 1),
                                     ("gelu_unrounded", 3), ("tanh_for_erf", 3), ("truncate", 0)])
def test_gemm_chain_rejects(bug, act, dtype):
    a, w, bias = _gemm_case(dtype, 24, 40, 256)
    if bug == "gelu_unrounded":  # pre-activations near zero, where the GELU slope is one half and the rounding shows
        bias = _rand(40, dtype=dtype, scale=0.05, seed=9)
    ch = G.gemm_chain(a, w, bias, act)
    _accepts(f"gemm act={act} without {bug}", _gemm_eager(a, w, bias, act), ch)
    _rejects(f"gemm act={act} {bug}", _gemm_eager(a, w, bias, act, bug), ch)


def _resid_eager(a, w, bias, resid, mod, mask, gate_row, B, T, S, bug=None):
    dt = a.dtype
    N = w.shape[0]
    y = (_acc(a, w) + bias.float()).to(dt).view(B, T, S, N)
    if gate_row < 0:
        return (resid.float().view(B, T, S, N) + y.float()).to(dt)
    m = mask
    if bug == "frame_late" and m is not None:
        m = torch.cat([m[:, :1], m[:, :-1]], 1)  # frame t takes frame t - 1's select
    gate = E._mod_row(mod, m, gate_row, B, T, N, dt).view(B, T, 1, N)
    g = gate.float() * y.float()
    if bug != "gate_unrounded":
        g = g.to(dt).float()
    return (resid.float().view(B, T, S, N) + g).to(dt)


def _resid_case(dtype):
    B, T, S, N, K = 2, 4, 3, 40, 128
    a, w, bias = _gemm_case(dtype, B * T * S, N, K)
    resid = _hidden(B * T * S, N, dtype=dtype, seed=7)
    mod = _rand(2, B, 6, N, dtype=dtype, scale=0.5, seed=8)
    mask = torch.tensor([[1, 0, 1, 1], [0, 1, 1, 0]], dtype=torch.uint8)
    return a, w, bias, resid, mod, mask, B, T, S


@both
@pytest.mark.parametrize("gate_row", [2, 5, -1])
def test_gemm_residual_chain_accepts_emulation(gate_row, dtype):
    a, w, bias, resid, mod, mask, B, T, S = _resid_case(dtype)
    for m in (None, mask):
        ch = G.gemm_residual_chain(a, w, bias, resid, mod, m, gate_row, B, T, S)
        _accepts(f"gemm residual gate_row={gate_row} mask={m is not None}", _resid_eager(a, w, bias, resid, mod, m, gate_row, B, T, S), ch)


@both
@pytest.mark.parametrize("bug", ["gate_unrounded", "frame_late"])
def test_gemm_residual_chain_rejects(bug, dtype):
    a, w, bias, resid, mod, mask, B, T, S = _resid_case(dtype)
    ch = G.gemm_residual_chain(a, w, bias, resid, mod, mask, 2, B, T, S)
    _rejects(f"gemm residual {bug}", _resid_eager(a, w, bias, resid, mod, mask, 2, B, T, S, bug), ch)


# ---------------------------------------------------------------------------------------------------------------------
# flash attention: the tiled online softmax in fp32, P 16-bit in the tile frame
# ---------------------------------------------------------------------------------------------------------------------
def _flash_eager(q, k, v, scale, lens, tile, bug=None):
    """q [nb, nq, H, D], k / v [nb, nk, H, D] -> [nb, nq, H, D] with the kernels' fp32 arithmetic."""
    nb, nq, H, D = q.shape
    nk = k.shape[1]
    dt = q.dtype
    if bug == "head_offset":
        q = torch.roll(q.reshape(nb, nq, H * D), -8, -1).view(nb, nq, H, D)
    sc = torch.tensor(scale, dtype=torch.float32)
    sl2 = sc if bug == "no_log2e" else sc * torch.tensor(G.LOG2E, dtype=torch.float32)
    L = [nk] * nb if lens is None else list(lens)
    if bug == "lens_shift":
        L = [L[0]] + L[:-1]
    L = [x + {"key_plus": 1, "key_minus": -1}.get(bug, 0) for x in L]
    out = torch.empty(nb, nq, H, D, dtype=dt)
    for b in range(nb):
        qh = q[b].permute(1, 0, 2).float()
        kh = k[b, :L[b]].permute(1, 0, 2).float()
        vh = v[b, :L[b]].permute(1, 0, 2).float()
        if bug == "final_frame":
            s = (qh @ kh.transpose(1, 2)) * sl2
            p = torch.exp2(s - s.amax(-1, keepdim=True))
            out[b] = ((p.to(dt).float() @ vh) * (1 / p.sum(-1, keepdim=True))).to(dt).permute(1, 0, 2)
            continue
        m = torch.full((H, nq, 1), -math.inf)
        l = torch.zeros(H, nq, 1)
        o = torch.zeros(H, nq, D)
        for k0 in range(0, L[b], tile):
            s = (qh @ kh[:, k0:k0 + tile].transpose(1, 2)) * sl2
            mx = torch.maximum(m, s.amax(-1, keepdim=True))
            a = torch.exp2(m - mx)
            p = torch.exp2(s - mx)
            P = p.to(dt).float()
            l = l * a + (P if bug == "l_rounded" else p).sum(-1, keepdim=True)
            o = (o if bug == "no_rescale" else o * a) + P @ vh[:, k0:k0 + tile]
            m = mx
        out[b] = (o * (1 / l)).to(dt).permute(1, 0, 2)
    return out


def _flash_case(dtype, D, nb=3, nq=24, nk=300, H=2, seed=0):
    g = _gen(seed)
    q = torch.randn(nb, nq, H, D, generator=g)
    q[..., 0] += 2.0
    k = torch.randn(nb, nk, H, D, generator=g)
    k[..., 0] += 3.0 * torch.arange(nk).view(1, nk, 1) / nk  # the max grows from tile to tile
    v = 0.3 + torch.randn(nb, nk, H, D, generator=g)
    return q.to(dtype), k.to(dtype), v.to(dtype), D**-0.5


@both
@pytest.mark.parametrize("D", [64, 32], ids=["tile128", "tile64"])
@pytest.mark.parametrize("lens", [None, [300, 129, 1]], ids=["full", "lens"])
def test_flash_chain_accepts_emulation(lens, D, dtype):
    q, k, v, scale = _flash_case(dtype, D)
    tile = G.tile_keys_of(D)
    ch = G.flash_chain(q, k, v, scale, lens)
    _accepts(f"flash D={D} lens={lens}", _flash_eager(q, k, v, scale, lens, tile), ch)


@both
@pytest.mark.parametrize("D", [64, 32], ids=["tile128", "tile64"])
@pytest.mark.parametrize("bug", ["key_plus", "key_minus", "lens_shift", "l_rounded", "final_frame", "no_rescale", "no_log2e",
                                 "head_offset"])
def test_flash_chain_rejects(bug, D, dtype):
    q, k, v, scale = _flash_case(dtype, D)
    lens = [257, 130, 65]  # last tiles partly filled, a key to spare behind each
    tile = G.tile_keys_of(D)
    ch = G.flash_chain(q, k, v, scale, lens)
    _rejects(f"flash D={D} {bug}", _flash_eager(q, k, v, scale, lens, tile, bug), ch)


@both
def test_flash_chain_row_subset(dtype):
    q, k, v, scale = _flash_case(dtype, 64, nb=1)
    rows = [0, 5, 23]
    sub = G.flash_chain(q, k, v, scale, rows=rows)
    _accepts("flash row subset", _flash_eager(q, k, v, scale, None, 128)[:, rows], sub)


# ---------------------------------------------------------------------------------------------------------------------
# attn_short: the eager chain
# ---------------------------------------------------------------------------------------------------------------------
def _rope_tables(n, D, seed=4):
    ang = torch.rand(n, D // 2, generator=_gen(seed)) * 6.0
    ang = ang.repeat_interleave(2, 1)
    return torch.cos(ang), torch.sin(ang)


def _short_eager(qkv, wq, wk, cos, sin, n, scale, flags, bug=None, eps=1e-6):
    rows, _, H, D = qkv.shape
    seqs = rows // n
    dt = qkv.dtype
    x = qkv.reshape(seqs, n, 3, H, D)
    q, k, v = x[:, :, 0], x[:, :, 1], x[:, :, 2]
    if n == 1:
        return v.clone()
    if not flags & 1:
        def rms(t, w):
            tf = t.float()
            return w * (tf * torch.rsqrt(tf.pow(2).mean(-1, keepdim=True) + eps)).to(dt)
        q, k = rms(q, wq), rms(k, wk)
    if cos is not None:
        pos = torch.arange(n).view(1, n, 1)
        if bug == "rope_pos":
            pos = (pos + 1) % n
        q, k = E._rope(q, cos, sin, pos), E._rope(k, cos, sin, pos)
    q, k, v = (t.transpose(1, 2).float() for t in (q, k, v))
    s32 = torch.tensor(scale, dtype=torch.float32)
    if flags & 2:
        p = ((q @ k.transpose(-1, -2)) * s32).softmax(-1)
    elif bug == "scale_after":
        p = ((q @ k.transpose(-1, -2)).to(dt).float() * s32).to(dt).float().softmax(-1)
    else:
        qs = (q * s32).to(dt).float()
        p = (qs @ k.transpose(-1, -2)).to(dt).float().softmax(-1)
    P = p if bug == "p_unrounded" else p.to(dt).float()
    return (P @ v).to(dt).transpose(1, 2)


def _short_case(dtype, n, D=72, H=2, seqs=3):
    qkv = _hidden(seqs * n, 3, H, D, dtype=dtype, seed=11)
    wq = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=12)
    wk = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=13)
    return qkv, wq, wk


@both
@pytest.mark.parametrize("flags", [0, 1, 3])
@pytest.mark.parametrize("rope", [False, True], ids=["plain", "rope"])
@pytest.mark.parametrize("n", [1, 2, 17, 33])
def test_short_chain_accepts_eager(n, rope, flags, dtype):
    D = 72 if n % 2 else 64
    qkv, wq, wk = _short_case(dtype, n, D)
    cos, sin = _rope_tables(n, D) if rope else (None, None)
    ch = G.short_chain(qkv, wq, wk, cos, sin, n, D**-0.5, flags, dtype)
    what = f"attn_short n={n} D={D} flags={flags} rope={rope}"
    _accepts(what, _short_eager(qkv, wq, wk, cos, sin, n, D**-0.5, flags), ch)
    if flags != 3:  # the stand-in of tests/kernels_emul.py (its SDPA is torch's, not the kernel's rounding)
        got = E.attn_short(qkv, wq, wk, cos, sin, 1, 3, 3 * n, n, 1, n, 2, D, D**-0.5, flags=flags)
        _accepts(what + " stand-in", got.view(3, n, 2, D), ch)


@both
@pytest.mark.parametrize("bug,flags,rope", [("scale_after", 0, False), ("p_unrounded", 0, False), ("p_unrounded", 3, False),
                                            ("rope_pos", 0, True), ("rope_pos", 3, True)])
def test_short_chain_rejects(bug, flags, rope, dtype):
    n, D = 20, 72  # D = 72: the scale is not a power of two, so where it is applied shows
    qkv, wq, wk = _short_case(dtype, n, D)
    cos, sin = _rope_tables(n, D) if rope else (None, None)
    ch = G.short_chain(qkv, wq, wk, cos, sin, n, D**-0.5, flags, dtype)
    _accepts(f"attn_short without {bug}", _short_eager(qkv, wq, wk, cos, sin, n, D**-0.5, flags), ch)
    _rejects(f"attn_short {bug}", _short_eager(qkv, wq, wk, cos, sin, n, D**-0.5, flags, bug), ch)
