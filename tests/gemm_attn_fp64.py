"""TEST INFRASTRUCTURE ONLY -- float64 reference chains of the GEMM (csrc/gemm_wgmma.cu) and attention kernels
(csrc/attn_wgmma.cu, csrc/attn_mma.cu, csrc/attn_short.cu), under the acceptance rule of tests/vae_fp64.py.

Each chain evaluates the real-valued core in float64, then the 16-bit rounding points the kernel comments name.  eps is
what the kernel's fp32 arithmetic can move a value by, derived below.  U32 = 2^-24 is the fp32 unit roundoff.

Accumulation on the tensor cores (wgmma, mma.sync).  Products of 16-bit values are exact in fp32; the sum of a K-term dot
product is off by the spread of an fp32 sum, sum_eps(sum of terms^2, K), and by the truncation of the fp32 partial sums:
the tensor cores round every k16 step's running sum towards zero, at most U32 |running sum| each.  conv_chain bounds that
by (K / 16) U32 |final value|, which assumes the partial sums are no larger than the final value.  A hidden-state A with a
DC offset against zero-mean W rows breaks that (the partial sums wander far from the final one), so `trunc_eps` takes the
partial sum after every k16 step in float64 (one rank-16 update per step, tiled over rows) and sums U32 |C_s|.  The
attention scores (D <= 128 terms, at most 8 k16 steps) use sum_i |terms| instead, which stays narrow there.

GEMM (gemm_chain, gemm_residual_chain)
  y = r(acc + bias):   eps = sum_eps + trunc_eps + U32 |acc + bias| (the fp32 add; none without bias).
  act 1, tanh-GELU:    gelu_tanh_f computes x / (1 + 2^w), w = x fma(x^2, kC1, kC0) -- x sigmoid(2u), which equals
                       torch's 0.5 x (1 + tanh u) exactly.  The two constants carry 2 and 3 fp32 roundings, x^2, the fma
                       and the product one each: |dw| <= 6 U32 (|kC0 x| + |kC1 x^3|).  ex2.approx is good to 2 ulp
                       (4 U32 relative) and moves 1 + e by ln2 |dw| e relatively; the add, rcp.approx (1 ulp) and the
                       final product add 4 U32.  With 1 - s = e / (1 + e), the relative bound is
                           rel = (1 - s) (ln2 |dw| + 4 U32) + 4 U32.
                       (The header's 5e-7 is absolute; this is the relative form the rule needs.)
                       Named widening, TANH_FLUSH_W: where w > 125 (x < -9.8) the reciprocal of 1 + 2^w is below 2^-126
                       and rcp.approx.ftz flushes it (and past w = 128 ex2 overflows to inf): the kernel returns -0.
                       The true value there is x 2^-w (|.| < 2^-121, a bf16 normal).  torch's fp32 tanh form returns 0
                       there too, by cancellation, so 0 is legal where any legal input has w > 125.  No absolute floor.
  act 3, erf-GELU:     gelu_erf_f is x * 0.5 * (1 + erff(x c)) in fp32: z = x c rounds twice (c and the product), erff
                       is good to 2 ulp, 1 + erf rounds, the last product rounds:
                           eps = 0.5 |x| (4 U32 |erf z| + erf'(z) 2 U32 |z| + U32 (1 + erf z)) + U32 |gelu|.
                       In the negative tail 1 + erf z cancels in fp32; the first term is the honest width of that.
  residual:            g = r(gate y) is exact in fp32 (eps 0); out = r(resid + g) as dit_fp64._add.

Flash attention (flash_chain), the attn_mma.cu header contract taken literally
  t_j = s_j scale log2e with s_j the float64 score, m_T the running max over the key tiles seen so far (128 keys for
  head_dim 64 / 72, 64 otherwise), p_j = 2^(t_j - m_T(j)) in the frame of its tile, P_j = r(p_j),
  O = sum P_j 2^(m_T(j) - m_last) v_j / sum p_j 2^(m_T(j) - m_last)   (l sums the unrounded p, as both kernels do).
  eps of t_j:   e_s = sum_eps(sum (q k)^2, D) + ceil(D / 16) U32 sum |q k|; e_t = |scale log2e| e_s + 3 U32 |t| (fp32(scale),
                its product with fp32(log2e), the product with the score).  The fp32 max differs from the float64 max by at
                most e_m = max_j e_t over the row.
  eps of p_j (relative):  d_j = ln2 (e_t + e_m + U32 |t - m|) + 4 U32 (exp2f and ex2.approx: 2 ulp each; the fp32
                subtraction).  P_j has both neighbours legal where p_j lies within d_j p_j of a midpoint.
                Named widening, P_FLUSH: ex2.approx.ftz (attn_wgmma) flushes 2^x < 2^-126 to zero, exp2f (attn_mma) keeps
                the subnormal; where p_j - d_j p_j < 2^-126 both are legal (this reaches bf16 only).
  eps of O, over l = sum p w (w = 2^(m_T - m_last)):
    spread of the ambiguous P_j:     sum (P_hi - P_lo) w |v| / l
    the fp32 P V sum:                sum_eps(sum (P w v)^2, L) / l + U32 sum_s |C_s| / l  (C_s: partial sums per k16 step)
    the fp32 l:                      |O| (sum_eps(sum (p w)^2, L) + sum d'_j p_j w_j) / l, d' = d without e_m: an error of
                                     the fp32 max scales every p of the frame and its P alike, so it cancels in O / l up
                                     to P's rounding, which the spread term holds
    the rescale where the max grows: 5 U32 (|C_b| + |O| l_b) / l at each tile boundary b whose tile max comes within 2 e_m
                                     of the running max (ex2 of a = exp2(m_old - m_new), and the products O a, l a + r; a
                                     itself is taken from the kernel's own fp32 maxima, the same for O and l)
    1 / l and the final multiply:    2 U32 |O|

attn_short (short_chain), the eager order of attn_short.cu and vsb200.h
  flags 0: y = RMSNorm (+ RoPE) of q, k (dit_fp64.qk_rmsnorm_chain), q' = r(q fp32(scale)) (one fp32 product: U32),
  S = r(q' k^T), p = softmax(S) in fp32, P = r(p), O = r(P V).  bit 0: no q / k norm.  bit 1: SDPA rounding -- fp32 scores
  times scale inside the softmax, r(p), r(P V).  n = 1 copies v.
  Scores of interval-valued q, k are bounded by interval products; e_S = sum_eps + ceil(D / 16) U32 sum |q k|.
  p_j rises with S_j and falls with every other S_k, so its bounds come from the corners: [exp(lo_j) / (exp(lo_j) +
  sum_k!=j exp(hi_k)), exp(hi_j) / (exp(hi_j) + sum_k!=j exp(lo_k))].  eps of p (relative): U32 |S - m| (fp32 subtraction)
  + 4 U32 (expf) + (n + 2) U32 (the n-term fp32 sum, 1 / d and the product).
  O: interval of sum P v from P's corners (v exact), eps = sum_eps(sum (P v)^2, n) + ceil(n / 16) U32 sum |P v|.

Everything is float64 arithmetic on exact 16-bit inputs and runs the same on the CPU and the GPU."""
import math

import torch

from tests.dit_fp64 import _add, mod_row, qk_rmsnorm_chain  # noqa: F401
from tests.vae_fp64 import U32, Chain, assert_legal, check, round16, sum_eps  # noqa: F401

LOG2E = 1.4426950408889634
LN2 = math.log(2.0)
TANH_FLUSH_W = 125.0  # w = -2 u log2e above which rcp.approx.ftz(1 + 2^w) flushes to zero
P_FLUSH = 2.0**-126   # smallest fp32 normal: ex2.approx.ftz returns 0 below it
_K0 = -2.0 * math.sqrt(2.0 / math.pi) * LOG2E  # kC0 of gelu_tanh_f (exact value; kC1 = 0.044715 kC0)


def _argmin(f, a=-2.0, b=0.0):
    """Turning point of a one-minimum function on [a, b] (golden-section search to float64 resolution)."""
    g = (math.sqrt(5) - 1) / 2
    for _ in range(200):
        c, d = b - g * (b - a), a + g * (b - a)
        if f(c) < f(d):
            b = d
        else:
            a = c
    return 0.5 * (a + b)


def gelu_tanh64(x):
    """0.5 x (1 + tanh(u)) = x sigmoid(2u), u = sqrt(2/pi) (x + 0.044715 x^3)."""
    w = _K0 * x * (1 + 0.044715 * x * x)  # -2 u log2e
    return x / (1 + torch.exp2(w))


def gelu_erf64(x):
    return x * 0.5 * (1 + torch.erf(x * math.sqrt(0.5)))


GELU_TANH_TURN = _argmin(lambda x: x / (1 + 2.0 ** (_K0 * x * (1 + 0.044715 * x * x))))
GELU_ERF_TURN = _argmin(lambda x: x * 0.5 * (1 + math.erf(x * math.sqrt(0.5))))


def gelu_tanh_eps(x):
    """eps of gelu_tanh_f at the float64 point x (module docstring)."""
    w = _K0 * x * (1 + 0.044715 * x * x)
    dw = 6 * U32 * (abs(_K0) * x.abs() + abs(_K0) * 0.044715 * x.abs() ** 3)
    one_minus_s = torch.sigmoid(w * LN2)  # e / (1 + e)
    return gelu_tanh64(x).abs() * (one_minus_s * (LN2 * dw + 4 * U32) + 4 * U32)


def gelu_erf_eps(x):
    z = x * math.sqrt(0.5)
    e = torch.erf(z)
    de = 2 / math.sqrt(math.pi) * torch.exp(-z * z)
    return 0.5 * x.abs() * (4 * U32 * e.abs() + de * 2 * U32 * z.abs() + U32 * (1 + e)) + U32 * gelu_erf64(x).abs()


# ---------------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------------
def _rows_chunk(M, N, budget=1 << 22):
    return max(1, min(M, budget // max(N, 1)))


def trunc_eps(a, w, step=16):
    """U32 sum_s |C_s| of a [M, K] @ w [N, K]^T: C_s the float64 partial sum after k16 step s (rows tiled)."""
    M, K = a.shape
    N = w.shape[0]
    out = torch.empty(M, N, dtype=torch.float64, device=a.device)
    wd = w.double()
    for r0 in range(0, M, _rows_chunk(M, N)):
        ad = a[r0:r0 + _rows_chunk(M, N)].double()
        c = torch.zeros(ad.shape[0], N, dtype=torch.float64, device=a.device)
        tot = torch.zeros_like(c)
        for k0 in range(0, K, step):
            c += ad[:, k0:k0 + step] @ wd[:, k0:k0 + step].T
            tot += c.abs()
        out[r0:r0 + ad.shape[0]] = tot
    return U32 * out


def acc_core(a, w):
    """(float64 a @ w^T, eps of its fp32 tensor-core accumulation)."""
    ad, wd = a.double(), w.double()
    acc = ad @ wd.T
    return acc, sum_eps((ad * ad) @ (wd * wd).T, a.shape[1]) + trunc_eps(a, w)


def gemm_linear_chain(a, w, bias):
    """y = r(a @ w^T + bias) of a [M, K], w [N, K]."""
    acc, e = acc_core(a, w)
    if bias is not None:
        acc = acc + bias.double()
        e = e + U32 * acc.abs()
    return Chain.start(acc, e, a.dtype)


def gemm_chain(a, w, bias, act):
    """out of gemm_bias_act (kernel epilogue numbering: 0 none, 1 tanh-GELU, 3 erf-GELU)."""
    y = gemm_linear_chain(a, w, bias)
    if act == 0:
        return y
    if act == 1:
        ch = y.step(gelu_tanh64, eps=gelu_tanh_eps(y.v), turn=GELU_TANH_TURN)
        flush = _K0 * y.lo * (1 + 0.044715 * y.lo * y.lo) > TANH_FLUSH_W  # TANH_FLUSH_W: the kernel may return -0
        ch.hi = torch.where(flush, torch.clamp_min(ch.hi, 0.0), ch.hi)
        return ch
    if act == 3:
        return y.step(gelu_erf64, eps=gelu_erf_eps(y.v), turn=GELU_ERF_TURN)
    raise ValueError(act)


def gemm_residual_chain(a, w, bias, resid, mod, mask, gate_row, B, T, S):
    """out of gemm_bias_residual: r(resid + r(gate y)) (gate_row >= 0, frame rows selected by mask) or r(resid + y)."""
    N = w.shape[0]
    y = gemm_linear_chain(a, w, bias)
    y = Chain(*(t.reshape(B, T, S, N) if t.dim() else t for t in (y.lo, y.hi, y.near, y.v, y.eps)), y.dtype)
    if gate_row >= 0:
        y = y.step(lambda yy, g: yy * g, mod_row(mod, mask, gate_row, B, T))
    return _add(y, resid.reshape(B, T, S, N))


# ---------------------------------------------------------------------------------------------------------------------
# flash attention
# ---------------------------------------------------------------------------------------------------------------------
def tile_keys_of(D):
    return 128 if D in (64, 72) else 64


def _flash_rows(qd, kd, vd, sl, tile, dtype):
    """(O, eps, P ambiguous count) for query rows qd [r, D] against keys kd, vd [L, D] (float64)."""
    L, D = kd.shape
    s = qd @ kd.T
    e_s = sum_eps((qd * qd) @ (kd * kd).T, D) + math.ceil(D / 16) * U32 * (qd.abs() @ kd.abs().T)
    t = s * sl
    e_t = abs(sl) * e_s + 3 * U32 * t.abs()
    e_m = e_t.amax(1, keepdim=True)
    nT = -(-L // tile)
    pad = nT * tile - L
    tp = torch.nn.functional.pad(t, (0, pad), value=-math.inf).view(-1, nT, tile)
    tmax = tp.amax(2)                                  # [r, nT]
    mrun = torch.cummax(tmax, 1).values               # running max after tile T
    mj = mrun.repeat_interleave(tile, 1)[:, :L]       # frame of each key
    m_last = mrun[:, -1:]
    x = t - mj
    p = torch.exp2(x)
    d = LN2 * (e_t + e_m + U32 * x.abs()) + 4 * U32
    ep = d * p
    P = round16(p, dtype)
    P_lo = torch.where(p - ep < P_FLUSH, torch.zeros_like(p), round16(p - ep, dtype))  # P_FLUSH
    P_hi = round16(p + ep, dtype)
    w = torch.exp2(mj - m_last)
    pw, Pw = p * w, P * w
    l = pw.sum(1, keepdim=True)
    O = (Pw @ vd) / l
    eps = ((P_hi - P_lo) * w) @ vd.abs() / l
    eps = eps + sum_eps((Pw * Pw) @ (vd * vd), L) / l
    # partial P V sums per k16 step (tiles are multiples of 16 keys, so the steps align with key 0)
    ns = -(-L // 16)
    Pw16 = torch.nn.functional.pad(Pw, (0, ns * 16 - L)).view(-1, ns, 16)
    v16 = torch.nn.functional.pad(vd, (0, 0, 0, ns * 16 - L)).view(ns, 16, D)
    C = torch.cumsum(torch.einsum("rsk,skd->rsd", Pw16, v16), 1)  # [r, ns, D]
    eps = eps + U32 * C.abs().sum(1) / l
    # the frame error e_m scales every p of a tile and its P alike, so it cancels in O / l (up to P's rounding, which
    # the spread term holds): the l term takes only the per-key part of d
    dl = LN2 * (e_t + U32 * x.abs()) + 4 * U32
    eps = eps + O.abs() * (sum_eps((pw * pw).sum(1, keepdim=True), L) + (dl * pw).sum(1, keepdim=True)) / l
    if nT > 1:
        grow = tmax[:, 1:] >= mrun[:, :-1] - 2 * e_m          # [r, nT - 1]: boundary after tile T
        lcum = torch.cumsum(pw, 1)
        bidx = torch.arange(1, nT, device=qd.device) * tile  # keys before the boundary
        Cb = C[:, bidx // 16 - 1]                             # [r, nT - 1, D]
        lb = lcum[:, bidx - 1]                                # [r, nT - 1]
        g = grow.double() * 5 * U32
        eps = eps + ((g.unsqueeze(2) * (Cb.abs() + O.abs().unsqueeze(1) * lb.unsqueeze(2))).sum(1)) / l
    eps = eps + 2 * U32 * O.abs()
    return O, eps, int((P_hi != P_lo).sum())


def flash_chain(q, k, v, scale, lens=None, tile_keys=None, rows=None, chunk=64):
    """Chain [nb, len(rows), H, D] of attn_flash on q [nb, nq, H, D], k / v [nb, nk, H, D] (any strides); lens: keys per
    batch; rows: the query rows to evaluate (default all), in chunks of `chunk` rows on q's device."""
    nb, nq, H, D = q.shape
    dt = q.dtype
    tile = tile_keys or tile_keys_of(D)
    rows = torch.arange(nq, device=q.device) if rows is None else torch.as_tensor(rows, device=q.device)
    sl = float(scale) * LOG2E
    O = torch.empty(nb, len(rows), H, D, dtype=torch.float64, device=q.device)
    E = torch.empty_like(O)
    amb = 0
    for b in range(nb):
        L = int(lens[b]) if lens is not None else k.shape[1]
        for h in range(H):
            kd, vd = k[b, :L, h].double(), v[b, :L, h].double()
            for r0 in range(0, len(rows), chunk):
                ri = rows[r0:r0 + chunk]
                o, e, a = _flash_rows(q[b, ri, h].double(), kd, vd, sl, tile, dt)
                O[b, r0:r0 + chunk, h], E[b, r0:r0 + chunk, h] = o, e
                amb += a
    ch = Chain.start(O, E, dt)
    ch.p_ambiguous = amb
    return ch


# ---------------------------------------------------------------------------------------------------------------------
# attn_short
# ---------------------------------------------------------------------------------------------------------------------
def _interval_dot(ql, qh, kl, kh):
    """Bounds of sum_d q_d k_d over q in [ql, qh], k in [kl, kh]: [.., n, D] x [.., n, D] -> [.., n, n]."""
    a, b = ql.unsqueeze(-2), qh.unsqueeze(-2)
    c, d = kl.unsqueeze(-3), kh.unsqueeze(-3)
    c1, c2, c3, c4 = a * c, a * d, b * c, b * d
    lo = torch.minimum(torch.minimum(c1, c2), torch.minimum(c3, c4)).sum(-1)
    hi = torch.maximum(torch.maximum(c1, c2), torch.maximum(c3, c4)).sum(-1)
    return lo, hi


def short_chain(qkv, wq, wk, cos, sin, n, scale, flags, dtype):
    """Chain [seqs, n, H, D] of attn_short on qkv [seqs * n, 3, H, D] (the sequences' token rows in order); cos / sin
    [n, D] fp32 tables or None; flags as vsb_attn_short."""
    rows, _, H, D = qkv.shape
    seqs = rows // n
    x = qkv.reshape(seqs, n, 3, H, D)
    if n == 1:
        return Chain.exact(x[:, :, 2])
    norm = (flags & 1) == 0
    sdpa = (flags & 2) != 0
    if norm or cos is not None:
        y = qk_rmsnorm_chain(qkv, wq if norm else None, wk if norm else None, H, D, rope_cos=cos, rope_sin=sin,
                             pos_div=1, pos_mod=n)
        y = Chain(*(t.reshape(seqs, n, 2, H, D) if t.dim() else t for t in (y.lo, y.hi, y.near, y.v, y.eps)), dtype)
    else:
        y = Chain.exact(x[:, :, :2])
    qn = Chain(*(t[:, :, 0] if t.dim() else t for t in (y.lo, y.hi, y.near, y.v, y.eps)), dtype)
    kn = Chain(*(t[:, :, 1] if t.dim() else t for t in (y.lo, y.hi, y.near, y.v, y.eps)), dtype)
    s32 = float(torch.tensor(scale, dtype=torch.float32))
    if not sdpa:
        qn = qn.step(lambda a: a * s32, eps=U32 * (qn.v * s32).abs())
    # [seqs, H, n, D]
    ql, qh, qc = (t.transpose(1, 2) for t in (qn.lo, qn.hi, qn.near))
    kl, kh, kc = (t.transpose(1, 2) for t in (kn.lo, kn.hi, kn.near))
    s_c = qc @ kc.transpose(-1, -2)
    s_lo, s_hi = _interval_dot(ql, qh, kl, kh)
    e_s = sum_eps((qc * qc) @ (kc * kc).transpose(-1, -2), D) + math.ceil(D / 16) * U32 * (qc.abs() @ kc.abs().transpose(-1, -2))
    if sdpa:  # fp32 scores times fp32(scale): one more rounding, and fp32(scale) is within U32 of scale
        lo, hi = (s_lo - e_s) * s32, (s_hi + e_s) * s32
        S_c, S_lo, S_hi = s_c * s32, lo - 2 * U32 * lo.abs(), hi + 2 * U32 * hi.abs()
    else:
        S_c, S_lo, S_hi = round16(s_c, dtype), round16(s_lo - e_s, dtype), round16(s_hi + e_s, dtype)
    M = S_hi.amax(-1, keepdim=True)
    eh, el = torch.exp(S_hi - M), torch.exp(S_lo - M)
    sh, sl_ = eh.sum(-1, keepdim=True), el.sum(-1, keepdim=True)
    p_lo = el / (el + (sh - eh).clamp_min(0))
    p_hi = eh / (eh + (sl_ - el).clamp_min(0))
    p = torch.softmax(S_c, -1)
    ep = p * (U32 * (S_c - S_c.amax(-1, keepdim=True)).abs() + 4 * U32 + (n + 2) * U32)
    P_lo, P_hi, P = round16(p_lo - ep, dtype), round16(p_hi + ep, dtype), round16(p, dtype)
    vd = x[:, :, 2].double().transpose(1, 2)  # [seqs, H, n, D]
    o_c = P @ vd
    o_lo = torch.minimum(P_lo.unsqueeze(-1) * vd.unsqueeze(-3), P_hi.unsqueeze(-1) * vd.unsqueeze(-3)).sum(-2)
    o_hi = torch.maximum(P_lo.unsqueeze(-1) * vd.unsqueeze(-3), P_hi.unsqueeze(-1) * vd.unsqueeze(-3)).sum(-2)
    e_o = sum_eps((P * P) @ (vd * vd), n) + math.ceil(n / 16) * U32 * (P @ vd.abs())
    T = lambda t: t.transpose(1, 2)  # noqa: E731  back to [seqs, n, H, D]
    return Chain(round16(T(o_lo - e_o), dtype), round16(T(o_hi + e_o), dtype), round16(T(o_c), dtype), T(o_c), T(e_o), dtype)


def legal_report(ch):
    """Print and return the fraction of elements with more than one legal value."""
    frac = float((ch.lo != ch.hi).double().mean())
    extra = f", {ch.p_ambiguous} ambiguous P" if hasattr(ch, "p_ambiguous") else ""
    print(f"    {100 * frac:.4f} % of the elements have more than one legal value{extra}")
    return frac
