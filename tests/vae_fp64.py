"""TEST INFRASTRUCTURE ONLY -- a float64 acceptance rule for the 16-bit VAE decoder kernels.

The reference of a kernel is the real-valued core of its operation (a convolution sum, GroupNorm statistics, a softmax,
an interpolation) evaluated in float64, followed by the reference model's own eager rounding points, each a cast to the
16-bit dtype.  At a rounding point the legal result is the nearest 16-bit value; where the float64 value lies within eps
of the midpoint between two 16-bit neighbours, both are legal, because the kernel's fp32 arithmetic may land on either
side.  So the legal set of one rounding point is [round(v - eps), round(v + eps)].  Chains carry that set as an interval
of 16-bit values: the next step is evaluated in float64 at the interval's corners (every step used here is monotone in
each chained argument, or names its one turning point), widened by its own eps and rounded outwards.  The kernel's
output must lie in the final interval, element by element.

eps is what the kernel's fp32 arithmetic can move the value by: for a K-term fp32 sum about 6 * sqrt(K) * 2^-24 *
sqrt(sum of terms^2), for a single fp32 operation a few fp32 ulps of the operands.

Everything here is exact float64 arithmetic on power-of-two scalings, so it runs the same on the CPU and the GPU."""
import math

import torch
import torch.nn.functional as F

U32 = 2.0**-24  # unit roundoff of fp32
# significand bits (with the implicit one), smallest normal exponent, largest exponent
_FMT = {torch.bfloat16: (8, -126, 127), torch.float16: (11, -14, 15)}


def fmt(dtype):
    return _FMT[dtype]


def max_finite(dtype):
    p, _, emax = _FMT[dtype]
    return (2.0 - 2.0 ** (1 - p)) * 2.0**emax


def ulp16(x, dtype):
    """Spacing of the 16-bit values at |x| (float64; subnormal spacing below the smallest normal)."""
    p, emin, _ = _FMT[dtype]
    x = x.double()
    _, e = torch.frexp(x)  # |x| = m * 2^e, m in [0.5, 1)
    e = torch.clamp(e.long() - 1, min=emin) - (p - 1)
    return ((e + 1023) << 52).view(torch.float64)  # 2^e built from its bits: exact on every device, unlike pow


def round16(x, dtype, mode="nearest"):
    """Round float64 x to the nearest 16-bit value, ties to even, exactly (no double rounding), returned as float64;
    mode="zero" truncates towards zero instead."""
    x = x.double()
    u = ulp16(x, dtype)
    q = x / u  # exact: u is a power of two
    r = (torch.round(q) if mode == "nearest" else torch.trunc(q)) * u
    big = r.abs() > max_finite(dtype)
    return torch.where(big, torch.copysign(torch.full_like(r, math.inf), r), r)


def sum_eps(sq_sum, K, c=6.0):
    """eps of a K-term fp32 sum whose terms have the given sum of squares."""
    return c * math.sqrt(K) * U32 * sq_sum.double().clamp_min(0).sqrt()


class Chain:
    """The legal 16-bit results [lo, hi] of a chain of rounding points, the all-nearest path `near`, and the float64
    value `v` and eps of the last rounding point (for the report)."""

    def __init__(self, lo, hi, near, v, eps, dtype):
        self.lo, self.hi, self.near, self.v, self.eps, self.dtype = lo, hi, near, v, eps, dtype

    @staticmethod
    def start(v, eps, dtype):
        """A first rounding point of the float64 core v."""
        v = v.double()
        eps = torch.as_tensor(eps, dtype=torch.float64, device=v.device)
        return Chain(round16(v - eps, dtype), round16(v + eps, dtype), round16(v, dtype), v, eps, dtype)

    @staticmethod
    def exact(x16):
        """A 16-bit tensor that is an input of the chain (one legal value)."""
        x = x16.double()
        return Chain(x, x, x, x, torch.zeros((), dtype=torch.float64, device=x.device), x16.dtype)

    def step(self, fn, *others, eps=0.0, turn=None):
        """Next rounding point r(fn(self, *others)).  Chains among `others` are expanded at their corners too; fn is
        monotone in each chained argument, except that a one-argument fn may have one turning point `turn` (its
        extremum), which is included when the interval straddles it."""
        args = [self, *others]
        ci = [i for i, a in enumerate(args) if isinstance(a, Chain)]
        center = fn(*[a.near if isinstance(a, Chain) else a for a in args])
        lo = hi = None
        for mask in range(1 << len(ci)):
            vals = list(args)
            for j, i in enumerate(ci):
                vals[i] = args[i].hi if mask >> j & 1 else args[i].lo
            val = fn(*vals)
            lo = val if lo is None else torch.minimum(lo, val)
            hi = val if hi is None else torch.maximum(hi, val)
        if turn is not None:
            assert not others
            inside = (self.lo < turn) & (self.hi > turn)
            ft = fn(torch.full_like(self.lo, turn))
            lo = torch.where(inside, torch.minimum(lo, ft), lo)
            hi = torch.where(inside, torch.maximum(hi, ft), hi)
        eps = torch.as_tensor(eps, dtype=torch.float64, device=center.device)
        return Chain(round16(lo - eps, self.dtype), round16(hi + eps, self.dtype), round16(center, self.dtype),
                     center, eps, self.dtype)

    def take(self, mask):
        f = lambda t: t.expand_as(self.near)[mask] if torch.is_tensor(t) and t.dim() else t  # noqa: E731
        return Chain(f(self.lo), f(self.hi), f(self.near), f(self.v), f(self.eps), self.dtype)


# ---------------------------------------------------------------------------------------------------------------------
# The reference chains of the decoder kernels.  Inputs are the kernels' own 16-bit (or fp32 statistics) tensors.
# ---------------------------------------------------------------------------------------------------------------------
SILU_TURN = -1.2784645427610738  # argmin of x * sigmoid(x)


def conv_chain(x, w, bias, resid=None, round_conv=True):
    """vae_conv3d of x [B, kt-1+T, H, W, Cin] with w [Cout, Cin, kt, 3, 3]: the float64 convolution (zero spatial
    padding), then r(r(conv) + bias) (round_conv, cuDNN's rounding) or r(conv + bias), then r(. + resid)."""
    dt = x.dtype
    xi = F.pad(x.permute(0, 4, 1, 2, 3).double(), (1, 1, 1, 1))
    wd = w.double()
    conv = F.conv3d(xi, wd).permute(0, 2, 3, 4, 1)
    sq = F.conv3d(xi * xi, wd * wd).permute(0, 2, 3, 4, 1)
    # wgmma accumulates in fp32 but rounds its partial sums towards zero, so besides the sqrt(K) spread of a K-term sum
    # its error has a bias that grows with the number of k16 accumulation steps
    K = w[0].numel()
    eps_sum = sum_eps(sq, K) + (K / 16) * U32 * conv.abs()
    b = bias.double()
    if round_conv:
        ch = Chain.start(conv, eps_sum, dt).step(lambda c, bb: c + bb, b, eps=U32 * (conv.abs() + b.abs()))
    else:
        ch = Chain.start(conv + b, eps_sum + U32 * (conv.abs() + b.abs()), dt)
    if resid is not None:
        r = resid.double()
        ch = ch.step(lambda y, rr: y + rr, r, eps=U32 * (ch.v.abs() + r.abs()))
    return ch


def gn_affine_chain(x, stats, gamma, beta):
    """n = r(a * x + b) of GroupNorm on x [B, ..., C] with the fp32 statistics [B, G, 2] (mean, rstd): torch keeps a
    16-bit input's mean and rstd in its dtype, a = rstd * gamma (exact in fp32), b = beta - a * mean and a * x + b in
    fp32 (two fp32 roundings)."""
    dt = x.dtype
    B, C, G = x.shape[0], x.shape[-1], stats.shape[1]
    shape = [B] + [1] * (x.dim() - 2) + [C]
    mean = round16(stats[..., 0].double(), dt).repeat_interleave(C // G, 1).view(shape)
    rstd = round16(stats[..., 1].double(), dt).repeat_interleave(C // G, 1).view(shape)
    a = rstd * gamma.double()
    ax, am, be = a * x.double(), a * mean, beta.double()
    v = ax + (be - am)
    return Chain.start(v, 2 * U32 * (ax.abs() + am.abs() + be.abs() + v.abs()), dt)


def silu64(s):
    return s / (1 + torch.exp(-s))


def sigmoid64(s):
    return 1 / (1 + torch.exp(-s))


def spatial_norm_silu_chain(n, zy, zb):
    """r(silu(r(r(n * zy) + zb))) with zy / zb already gathered to n's shape (16-bit).  n * zy of two 16-bit values is
    exact in fp32; the add rounds once in fp32; silu is x / (1 + expf(-x)) in fp32."""
    m = n.step(lambda a, b: a * b, zy.double())
    zbd = zb.double()
    s = m.step(lambda a, b: a + b, zbd, eps=U32 * (m.v.abs() + zbd.abs()))
    # below about -88, expf(-x) overflows fp32 and x / (1 + inf) is -0, in the kernel and in torch's fp32 silu alike:
    # where any legal input is below -80 (|silu| < 2e-33) the result may be anything down to zero
    fp32_range = torch.where(s.lo < -80, torch.full_like(s.v, 2.0**-100), torch.zeros_like(s.v))
    return s.step(silu64, eps=6 * U32 * silu64(s.v).abs() + fp32_range, turn=SILU_TURN)


def sigmoid_act_chain(n):
    """r(n * r(sigmoid(n))): torch.sigmoid in fp32 (rounded), then the 16-bit product (exact in fp32, rounded once)."""
    sig = n.step(sigmoid64, eps=4 * U32 * sigmoid64(n.v))
    return n.step(lambda a, b: a * b, sig)


def check(what, got, chain, mask=None, verbose=True):
    """Report and return (ok, stats) of the 16-bit kernel output `got` against the legal set of `chain`: bit-equal
    fraction (to the all-nearest path), largest error in ulps, largest |v - midpoint| of an accepted flip and its eps."""
    g = got.double()
    c = chain
    if mask is not None:
        g, c = g[mask], chain.take(mask)
    near = c.near.expand_as(g)
    lo, hi = c.lo.expand_as(g), c.hi.expand_as(g)
    both_nan = torch.isnan(g) & torch.isnan(near)
    inside = ((g >= lo) & (g <= hi)) | both_nan
    equal = (g == near) | both_nan
    n = g.numel()
    diff = (g - near).abs()
    finite = torch.isfinite(diff)
    ulps = torch.where(finite, diff / ulp16(torch.maximum(g.abs(), near.abs()), c.dtype), torch.zeros_like(diff))
    ulps = torch.where(finite | equal, ulps, torch.full_like(ulps, math.inf))
    flips = inside & ~equal
    mid_dist = (c.v.expand_as(g) - 0.5 * (g + near)).abs()
    eps = c.eps.expand_as(g)
    st = dict(n=n, bit_equal=float(equal.double().mean()) if n else 1.0, max_ulp=float(ulps.max()) if n else 0.0,
              flips=int(flips.sum()), bad=int((~inside).sum()),
              max_flip_mid=float(mid_dist[flips].max()) if bool(flips.any()) else 0.0,
              eps_at_flip=float(eps[flips][mid_dist[flips].argmax()]) if bool(flips.any()) else 0.0,
              max_eps=float(eps.max()) if n else 0.0)
    if verbose:
        print(f"[{what}] n={n} eps<={st['max_eps']:.3g}: bit-equal {100 * st['bit_equal']:.4f} %, max {st['max_ulp']:.0f} ulp, "
              f"{st['flips']} accepted flips (largest |v - mid| {st['max_flip_mid']:.3g} at eps {st['eps_at_flip']:.3g}), "
              f"{st['bad']} outside the legal set")
        if st["bad"]:
            idx = (~inside).nonzero()[:6]
            for i in idx:
                i = tuple(int(a) for a in i)
                print(f"    at {i}: got {float(g[i]):.9g}, legal [{float(lo[i]):.9g}, {float(hi[i]):.9g}], "
                      f"float64 {float(c.v.expand_as(g)[i]):.9g}")
    return st["bad"] == 0, st


def assert_legal(what, got, chain, mask=None):
    ok, st = check(what, got, chain, mask)
    assert ok, f"{what}: {st['bad']} of {st['n']} elements outside the legal set"
    return st


def assert_bit_exact(what, got, want):
    """Pure data movement: identical bits (NaN payloads included)."""
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape)
    g, w = got.contiguous().view(torch.int16), want.contiguous().view(torch.int16)
    bad = int((g != w).sum())
    print(f"[{what}] n={g.numel()}: bit-exact {100 * (1 - bad / max(g.numel(), 1)):.4f} %")
    assert bad == 0, f"{what}: {bad} elements differ"
