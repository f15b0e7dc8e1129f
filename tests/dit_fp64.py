"""TEST INFRASTRUCTURE ONLY -- float64 reference chains of the transformer-block kernels (csrc/elementwise.cu,
csrc/dwconv.cu, csrc/patch_embed.cu), under the acceptance rule of tests/vae_fp64.py.

One function per kernel.  Each evaluates the real-valued core of the operation in float64 and then the 16-bit rounding
points of the reference model's eager code, which the kernel comments name.  A chain whose every eps is zero (products
and sums of two 16-bit values are exact in fp32, so the one rounding is the correctly rounded one) has exactly one legal
result: those functions return a 16-bit tensor to compare bit for bit.  The others return a `Chain`.

eps of the normalisations (`ln_core`, `qk_rmsnorm_chain`): the kernels take two-pass statistics in fp32.
  * mean: an fp32 sum of the C 16-bit inputs (exact terms), so off by about sum_eps(sum x^2, C), divided by C, one more
    rounding for the division:                      dm   = sum_eps(sum x^2, C) / C + U32 |mean|
  * variance: sum (x - m')^2 / C = var + (m' - mean)^2 exactly, each d = x - m' and d * d rounded (3 roundings per term),
    an fp32 sum of C terms, the division and the + eps:
                                                    dvar = dm^2 + (sum_eps(sum d^4, C) + 4 U32 sum d^2) / C + 2 U32 (var + eps)
  * rsqrtf is good to 2 ulp = 4 U32, and d rstd / d var = -rstd / (2 (var + eps)):
                                                    rel  = dvar / (2 (var + eps)) + 4 U32
  * n = (x - m') * rstd' with two roundings:        en   = dm rstd + |n| (rel + 2 U32)
  * the affine form n * gamma + beta adds two roundings (one if fused): en |gamma| + 2 U32 (|n gamma| + |n gamma + beta|)
n is not monotone in the statistics in a way Chain.step handles, so a chain starts at n with this eps.  On a row with a
large offset and a small spread dm * rstd dominates and the legal interval is honestly wide: that is how far fp32
two-pass statistics can be from float64 there.  (A constant row is the exception: every partial sum k * x is exact in
fp32, so n is exactly zero; the GPU tests pin that separately.)

Everything is float64 arithmetic on exact inputs and runs the same on the CPU and the GPU."""
import torch
import torch.nn.functional as F

from tests.vae_fp64 import (U32, Chain, assert_bit_exact, assert_legal, check, round16, sum_eps,  # noqa: F401
                            ulp16)


def to16(v, dtype):
    """A float64 tensor of 16-bit values as that dtype (exact)."""
    return v.to(dtype)


def _add(ch, t):
    """r(ch + t) computed as an fp32 add followed by the cast (the sum of two 16-bit values is exact in fp32 unless their
    exponents are far apart; then the fp32 rounding moves it by at most U32 |sum|)."""
    t = t.double()
    return ch.step(lambda a, b: a + b, t, eps=U32 * (ch.v + t).abs())


# ---------------------------------------------------------------------------------------------------------------------
# modulation table, LayerNorm + modulate, gate + residual
# ---------------------------------------------------------------------------------------------------------------------
def modulation_table_ref(table, t, t0):
    """mod[s, b, r, c] = r(table[r, c] + (s ? t0 : t)[b, r * C + c]); without t0 both halves are the t rows."""
    rows, C = table.shape
    B = t.shape[0]
    m0 = round16(table.double()[None] + t.double().view(B, rows, C), table.dtype)
    m1 = m0 if t0 is None else round16(table.double()[None] + t0.double().view(B, rows, C), table.dtype)
    return to16(torch.stack([m0, m1]), table.dtype)


def mod_row(mod, mask, row, B, T):
    """Row `row` of mod [2, B, R, C] per frame as float64 [B, T, 1, C]: the t rows where mask[b, t] != 0 (or no mask),
    the t0 rows where it is zero."""
    m = mod.double()
    C = m.shape[-1]
    r0 = m[0, :, row].view(B, 1, 1, C).expand(B, T, 1, C)
    if mask is None:
        return r0
    r1 = m[1, :, row].view(B, 1, 1, C).expand(B, T, 1, C)
    return torch.where(mask.view(B, T, 1, 1) != 0, r0, r1)


def ln_core(x, eps, gamma=None, beta=None, delta=None):
    """(v, e) of LayerNorm over the last dimension of x: v = (x - mean) * rstd [* gamma + beta] in float64 with the biased
    variance, e as derived in the module docstring.  delta >= 0: x itself is only known to +- delta (a 16-bit intermediate
    with more than one legal value); e then also holds the first-order sensitivity of n to that:
    |dn_i| <= rstd (delta_i + sum delta / C) + |n_i| dvar' / (2 (var + eps)),  dvar' = (2 sum delta |d| + sum delta^2) / C."""
    x = x.double()
    C = x.shape[-1]
    mean = x.mean(-1, keepdim=True)
    d = x - mean
    var = (d * d).mean(-1, keepdim=True)
    ve = var + eps
    rstd = ve.rsqrt()
    dm = sum_eps((x * x).sum(-1, keepdim=True), C) / C + U32 * mean.abs()
    dvar = dm * dm + (sum_eps((d ** 4).sum(-1, keepdim=True), C) + 4 * U32 * (d * d).sum(-1, keepdim=True)) / C + 2 * U32 * ve
    n = d * rstd
    e = dm * rstd + n.abs() * (dvar / (2 * ve) + 6 * U32)
    if delta is not None:
        dv2 = (2 * (delta * d.abs()).sum(-1, keepdim=True) + (delta * delta).sum(-1, keepdim=True)) / C
        e = e + rstd * (delta + delta.sum(-1, keepdim=True) / C) + n.abs() * dv2 / (2 * ve)
    if gamma is None:
        return n, e
    g, b = gamma.double(), beta.double()
    v = n * g + b
    return v, e * g.abs() + 2 * U32 * ((n * g).abs() + v.abs())


def ln_modulate_chain(x, mod, mask, shift_row, scale_row, B, T, S, eps=1e-6, gamma=None, beta=None):
    """n = r(LN(x)) (with gamma / beta: one rounding after weight and bias); g = r(1 + scale); m = r(n * g);
    out = r(m + shift), rows of mod selected per frame by mask.  Only n has eps > 0.  Shape [B, T, S, C]."""
    C = x.shape[-1]
    v, e = ln_core(x.reshape(B, T, S, C), eps, gamma, beta)
    n = Chain.start(v, e, x.dtype)
    g = round16(1.0 + mod_row(mod, mask, scale_row, B, T), x.dtype)
    m = n.step(lambda a, b: a * b, g)
    return m.step(lambda a, b: a + b, mod_row(mod, mask, shift_row, B, T))


def gate_residual_ref(x, y, mod, mask, gate_row, B, T, S):
    """(cache, out) = (r(gate * y), r(x + cache)) as 16-bit tensors of x's shape; both operations are exact before their
    rounding."""
    C = x.shape[-1]
    g = round16(mod_row(mod, mask, gate_row, B, T) * y.double().reshape(B, T, S, C), x.dtype)
    out = round16(x.double().reshape(B, T, S, C) + g, x.dtype)
    return to16(g, x.dtype).reshape(x.shape), to16(out, x.dtype).reshape(x.shape)


def residual_add_ref(x, y):
    return to16(round16(x.double() + y.double().reshape(x.shape), x.dtype), x.dtype)


def unshuffle_index(B, T, H, W, down, device="cpu"):
    """For every token row (b, t, h, w) of the natural order, its row in the sub-grid order
    [(b dt dh dw), (t/dt h/dh w/dw)] of dwconv_shuffle (DownSampler.reverse reads y there)."""
    dt, dh, dw = down
    b, t, h, w = torch.meshgrid(*(torch.arange(n, device=device) for n in (B, T, H, W)), indexing="ij")
    sub = ((b * dt + t % dt) * dh + h % dh) * dw + w % dw
    tok = ((t // dt) * (H // dh) + h // dh) * (W // dw) + w // dw
    return (sub * ((T // dt) * (H // dh) * (W // dw)) + tok).reshape(-1)


def gate_residual_unshuffle_ref(x, y, mod, gate_row, B, T, H, W, down):
    C = x.shape[-1]
    yn = y.reshape(-1, C)[unshuffle_index(B, T, H, W, down, x.device)].reshape(B, T * H * W, C)
    return gate_residual_ref(x.reshape(B, T * H * W, C), yn, mod, None, gate_row, B, 1, T * H * W)[1].reshape(x.shape)


# ---------------------------------------------------------------------------------------------------------------------
# q / k normalisation and RoPE on the packed [rows, 3, H, D] buffer
# ---------------------------------------------------------------------------------------------------------------------
def _positions(rows, pos_div, pos_mod, device):
    return (torch.arange(rows, device=device) // pos_div) % pos_mod


def _rot_pairs(ch):
    """rotate_half on interleaved pairs as a chain: rot[2i] = -y[2i + 1], rot[2i + 1] = y[2i]."""
    def rot(a, b):  # a supplies the odd elements (negated), b the even ones
        return torch.stack((-a[..., 1::2], b[..., 0::2]), -1).flatten(-2)
    return Chain(rot(ch.hi, ch.lo), rot(ch.lo, ch.hi), rot(ch.near, ch.near), rot(ch.v, ch.v), ch.eps, ch.dtype)


def qk_rmsnorm_chain(qkv, wq, wk, H, D, eps=1e-6, rope_cos=None, rope_sin=None, pos_div=1, pos_mod=1):
    """The q and k thirds [rows, 2, H, D] of qk_rmsnorm_: h = r(x * rsqrt(mean(x^2) + eps)), y = r(w * h); with fp32
    tables then r(y * cos + rot(y) * sin) at position (row // pos_div) % pos_mod; wq = wk = None is RoPE alone.
    eps of h: the squares are exact in fp32, their D-term sum is off by sum_eps(sum x^4, D), the division and the + eps
    round (2 U32), rsqrtf is 4 U32, the product x * rstd rounds once.  eps of the rotation: two fp32 products and one fp32
    add, each within U32 of its result (twice that is allowed)."""
    dt = qkv.dtype
    rows = qkv.numel() // (3 * H * D)
    x16 = qkv.reshape(rows, 3, H, D)[:, :2]
    if wq is not None:
        x = x16.double()
        ve = (x * x).mean(-1, keepdim=True) + eps
        dms = sum_eps((x ** 4).sum(-1, keepdim=True), D) / D + 2 * U32 * ve
        v = x * ve.rsqrt()
        h = Chain.start(v, v.abs() * (dms / (2 * ve) + 5 * U32), dt)
        y = h.step(lambda a, b: a * b, torch.stack([wq, wk]).double().view(1, 2, 1, D))
    else:
        y = Chain.exact(x16)
    if rope_cos is None:
        return y
    pos = _positions(rows, pos_div, pos_mod, qkv.device)
    c, s = rope_cos.double()[pos].view(rows, 1, 1, D), rope_sin.double()[pos].view(rows, 1, 1, D)
    rot = _rot_pairs(y)
    e = 2 * U32 * ((y.near * c).abs() + (rot.near * s).abs() + (y.near * c + rot.near * s).abs())
    return y.step(lambda a, b, cc, ss: a * cc + b * ss, rot, c, s, eps=e)


def qk_layernorm_chain(qkv, wq, bq, wk, bk, H, D, eps=1e-6):
    """The q and k thirds of qk_layernorm_: r(((x - mean) * rstd) * w + b) per head."""
    rows = qkv.numel() // (3 * H * D)
    g = torch.stack([wq, wk]).view(1, 2, 1, D)
    b = torch.stack([bq, bk]).view(1, 2, 1, D)
    return Chain.start(*ln_core(qkv.reshape(rows, 3, H, D)[:, :2], eps, g, b), qkv.dtype)


def qk_rope_halves_ref(qkv, rope_cos, rope_sin_signed, H, D, half, pos_div=1, pos_mod=1):
    """qk_rope_halves_ as a 16-bit tensor [rows, 3, H, D]: r(r(t * cos) + r(partner * sin)) on q and k, partner = the other
    half of the element's block of 2 * half channels, the tables holding 16-bit values (so every product and the sum are
    exact before their rounding); v unchanged."""
    dt = qkv.dtype
    rows = qkv.numel() // (3 * H * D)
    v = qkv.reshape(rows, 3, H, D)
    t = v[:, :2].double()
    pos = _positions(rows, pos_div, pos_mod, qkv.device)
    c, s = rope_cos.double()[pos].view(rows, 1, 1, D), rope_sin_signed.double()[pos].view(rows, 1, 1, D)
    partner = t.reshape(rows, 2, H, D // (2 * half), 2, half).flip(4).reshape(rows, 2, H, D)
    out = round16(round16(t * c, dt) + round16(partner * s, dt), dt)
    return torch.cat([to16(out, dt), v[:, 2:]], 1)


def assert_qk(what, got, orig, chain):
    """q and k of the updated buffer inside the chain's legal set, v bit-identical to the input's."""
    H, D = chain.near.shape[-2:]
    g, o = got.reshape(-1, 3, H, D), orig.reshape(-1, 3, H, D)
    st = assert_legal(what, g[:, :2], chain)
    assert_bit_exact(what + " v untouched", g[:, 2].contiguous(), o[:, 2].contiguous())
    return st


# ---------------------------------------------------------------------------------------------------------------------
# depth-wise convolutions
# ---------------------------------------------------------------------------------------------------------------------
def _tap_sums(taps):
    """float64 (sum, sum of squares, sum of magnitudes) of an iterable of per-tap product tensors."""
    s = q = a = None
    for t in taps:
        s, q, a = (t, t * t, t.abs()) if s is None else (s + t, q + t * t, a + t.abs())
    return s, q, a


def _conv_start(taps, K, dtype, lead=None):
    """First rounding point of a K-tap fp32 fma chain (+ lead, a term that enters the fp32 sum first)."""
    s, q, a = _tap_sums(taps)
    if lead is not None:
        s, q, a = s + lead, q + lead * lead, a + lead.abs()
    return Chain.start(s, sum_eps(q, K) + 2 * U32 * a, dtype)


def _same_taps(x5, w_taps, ksize):
    """Per-tap products of the depth-wise conv with zero "same" padding: x5 [B, T, H, W, C], w_taps [kt*kh*kw, C]."""
    kt, kh, kw = ksize
    B, T, H, W, C = x5.shape
    xp = F.pad(x5.double(), (0, 0, kw // 2, kw // 2, kh // 2, kh // 2, kt // 2, kt // 2))
    w = w_taps.double()
    for a in range(kt):
        for b in range(kh):
            for c in range(kw):
                yield xp[:, a:a + T, b:b + H, c:c + W] * w[(a * kh + b) * kw + c]


def dwconv_chain(x, w_taps, bias, B, T, H, W, ksize):
    """dwconv_shuffle before its permutation, [B, T, H, W, C]: r(r(r(conv) + bias) + x)."""
    C = x.shape[-1]
    x5 = x.reshape(B, T, H, W, C)
    ch = _conv_start(_same_taps(x5, w_taps, ksize), w_taps.shape[0], x.dtype)
    return _add(_add(ch, bias), x5)


def shuffle_rows(t, B, T, H, W, down):
    """[B, T, H, W, C] -> [(b dt dh dw), (t/dt h/dh w/dw), C], the order dwconv_shuffle stores in."""
    dt, dh, dw = down
    C = t.shape[-1]
    v = t.reshape(B, T // dt, dt, H // dh, dh, W // dw, dw, C)
    return v.permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(B * dt * dh * dw, -1, C)


def dwconv_ffn_chain(h, w_taps, bias, BT, H, W):
    """out = r(r(r(h + c5) + c3) + c1), ck = r(r(conv_k(h)) + bias_k): the eager out = out + module(x) per kernel size."""
    C = h.shape[-1]
    x5 = h.reshape(BT, 1, H, W, C)
    b = bias.double()
    c5 = _add(_conv_start(_same_taps(x5, w_taps[:25], (1, 5, 5)), 25, h.dtype), b[0])
    c3 = _add(_conv_start(_same_taps(x5, w_taps[25:34], (1, 3, 3)), 9, h.dtype), b[1])
    c1 = _add(Chain.start(x5.double() * w_taps[34].double(), 0.0, h.dtype), b[2])  # one exact product
    add = lambda p, q: p + q  # noqa: E731
    s = _add(c5, x5)
    s = s.step(add, c3, eps=U32 * (s.v + c3.v).abs())
    return s.step(add, c1, eps=U32 * (s.v + c1.v).abs())


def kv_compress_chain(x, w_taps, bias, ln_w, ln_b, B, T, H, W, window, pad_t=0, eps=1e-5, round_conv=True):
    """[B, Tc, Hc, Wc, C]: the depth-wise conv with stride = window after pad_t leading copies of frame 0 (rows / columns /
    frames past the last whole window unread); y = r(r(conv) + bias) (round_conv) or r(bias + conv); then
    r(LN(y) * ln_w + ln_b).  The statistics are those of the all-nearest y; on the rare elements where y has two legal
    values the LayerNorm eps carries the sensitivity to them (ln_core's delta); an accepted flip on such an element is the
    other legal y carried through, so it sits near that eps by construction.  Returns (chain, chain of y)."""
    C = x.shape[-1]
    kt, kh, kw = window
    v = x.reshape(B, T, H, W, C).double()
    if pad_t:
        v = torch.cat([v[:, :1].expand(B, pad_t, H, W, C), v], 1)
    Tc, Hc, Wc = (T + pad_t) // kt, H // kh, W // kw
    w = w_taps.double()
    taps = (v[:, a::kt][:, :Tc, b::kh][:, :, :Hc, c::kw][:, :, :, :Wc] * w[(a * kh + b) * kw + c]
            for a in range(kt) for b in range(kh) for c in range(kw))
    if round_conv:
        y = _add(_conv_start(taps, kt * kh * kw, x.dtype), bias)
    else:
        y = _conv_start(taps, kt * kh * kw + 1, x.dtype, lead=bias.double().expand(B, Tc, Hc, Wc, C))
    return Chain.start(*ln_core(y.near, eps, ln_w, ln_b, delta=y.hi - y.lo), x.dtype), y


def patch_embed_chain(z, weight, bias, pos, ph, pw):
    """[B, T, S, C] tokens of z [B, Cin, T, H, W]: the (1, ph, pw)-strided conv of the zero-padded latent (16 taps in the
    order (c, dy, dx)), r(conv), r(. + bias), r(. + pos)."""
    B, Cin, T, H, W = z.shape
    C = weight.shape[0]
    Hn, Wn = -(-H // ph), -(-W // pw)
    zp = F.pad(z.double(), (0, Wn * pw - W, 0, Hn * ph - H))
    p = zp.view(B, Cin, T, Hn, ph, Wn, pw).permute(0, 2, 3, 5, 1, 4, 6).reshape(B, T, Hn * Wn, 1, Cin * ph * pw)
    w = weight.double().reshape(1, 1, 1, C, Cin * ph * pw)
    K = Cin * ph * pw
    ch = _conv_start((p[..., k] * w[..., k] for k in range(K)), K, z.dtype)
    if bias is not None:
        ch = _add(ch, bias)
    return _add(ch, pos) if pos is not None else ch
