"""Thin torch-tensor front end of the C-ABI (videosys_b200/_lib.py): pointer + shape marshalling only.

Every function enqueues exactly one sm_90a kernel on the current CUDA stream (capturable in a CUDA graph).  CPU tensors are rejected:
there is no fallback path.
"""
import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib

_initialised = set()

# bench.py sets this to a list to time individual launches with CUDA events on the launching stream:
# entries are (kind, start_event, end_event, algorithmic_work) -- work = FLOPs for gemm/attn, bytes otherwise.
# PROFILE_KINDS (a set, or None for every kind) limits which launches carry events: inside bench.py's timed region
# only the dominant kernel does, so the measurement itself costs < 1 % (2 events x 3472 launches cost ~1 % of a step).
PROFILE = None
PROFILE_KINDS = None


class _Timed:
    __slots__ = ("kind", "work", "e0", "cancelled")

    def __init__(self, kind, work):
        self.kind, self.work = kind, work
        self.cancelled = False

    def __enter__(self):
        self.e0 = None
        if PROFILE is not None and (PROFILE_KINDS is None or self.kind in PROFILE_KINDS):
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def cancel(self):
        """Nothing was launched inside this block: record no entry."""
        self.cancelled = True

    def __exit__(self, *exc):
        if self.e0 is not None and not self.cancelled:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            PROFILE.append((self.kind, self.e0, e1, self.work))
        return False


def _init_dev(lib, dev):
    if dev not in _initialised:
        _lib.check(lib.vsb_init(dev), "init")
        _initialised.add(dev)


def _prep(*tensors):
    lib = _lib.load()
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise _lib.VsbError("vsb200 kernels need CUDA tensors (no CPU fallback)")
        if not t.is_contiguous():
            raise _lib.VsbError("vsb200 kernels need contiguous tensors")
        dev = t.device.index if dev is None else dev
    _init_dev(lib, dev)
    return lib, torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def require_cuda(t, what: str = "vsb200", half_only: bool = False):
    """The model front ends call this first: there is no CPU execution path (and the kernels take 16-bit activations)."""
    if not t.is_cuda:
        raise RuntimeError(f"videosys_b200 {what} runs on sm_90a CUDA devices only (no CPU path)")
    if half_only and t.dtype not in (torch.bfloat16, torch.float16):
        raise RuntimeError(f"videosys_b200 {what} runs in fp16 / bf16 only")


def _bf16(t, name):
    if t is not None and t.dtype not in (torch.bfloat16, torch.float16):
        raise _lib.VsbError(f"{name} must be bfloat16 or float16")


def _fn(lib, name, ref):
    """The entry for ref's dtype: bf16 -> `name`, IEEE fp16 -> its twin `name_f16` (include/vsb200.h)."""
    if ref.dtype == torch.float16:
        return getattr(lib, name + "_f16")
    if ref.dtype != torch.bfloat16:
        raise _lib.VsbError(f"vsb200 kernels take bfloat16 or float16 tensors, got {ref.dtype}")
    return getattr(lib, name)


def _same_dtype(*tensors):
    dt = None
    for t in tensors:
        if t is None or not t.dtype.is_floating_point or t.dtype == torch.float32:
            continue
        if dt is None:
            dt = t.dtype
        elif t.dtype != dt:
            raise _lib.VsbError(f"vsb200 kernels need one 16-bit dtype per call, got {dt} and {t.dtype}")


def set_option(name: str, value: int) -> None:
    _lib.check(_lib.load().vsb_set_option(name.encode(), int(value)), "set_option")


def launch_count() -> int:
    return int(_lib.load().vsb_launch_count())


# kernels executed by replaying captured CUDA graphs (core/graph_step.py adds a graph's launch count on every replay
# after the first; the first replay's launches were counted by vsb_launch_count at capture time)
GRAPH_REPLAYED_LAUNCHES = 0


def executed_launch_count() -> int:
    """Kernels of this library that have run: host launches + launches inside replayed CUDA graphs."""
    return launch_count() + GRAPH_REPLAYED_LAUNCHES


def tmap_cache_stats():
    """(hits, misses) of the encoded-tensor-map cache; misses = host cuTensorMapEncodeTiled calls made."""
    lib = _lib.load()
    return int(lib.vsb_tmap_cache_stats(0)), int(lib.vsb_tmap_cache_stats(1))


def modulation_table(table: torch.Tensor, t: torch.Tensor, t0: Optional[torch.Tensor]) -> torch.Tensor:
    """[2, B, rows, C] = table + t (and + t0); rows = table.shape[0] (6 for blocks, 2 for the final layer)."""
    lib, st = _prep(table, t, t0)
    rows, Cc = table.shape
    B = t.shape[0]
    _same_dtype(table, t, t0)
    mod = torch.empty(2, B, rows, Cc, dtype=table.dtype, device=table.device)
    _lib.check(_fn(lib, "vsb_modulation_table", table)(_p(table), _p(t), _p(t0), _p(mod), B, Cc, rows, st), "modulation_table")
    return mod


def patch_embed(z, weight, bias, pos, ph: int, pw: int, s0: int = 0, s_local: Optional[int] = None):
    """Tokens [B, T, S_local, C] of a latent z [B, Cin, T, H, W] (contiguous): the (1, ph, pw)-strided patch convolution
    (weight = conv.weight, any [C, Cin, (1,) ph, pw] shape), + bias, + pos [S, C], for patch columns s0 .. s0+S_local-1
    (columns beyond the grid are zero).  Returns None when the kernel does not take the shape (Cin*ph*pw != 16)."""
    lib, st = _prep(z, weight, bias, pos)
    _bf16(z, "z")
    _same_dtype(z, weight, bias, pos)
    B, Cin, T, H, W = z.shape
    Cc = weight.shape[0]
    S = -(-H // ph) * -(-W // pw)
    s_local = S if s_local is None else s_local
    out = torch.empty(B, T, s_local, Cc, dtype=z.dtype, device=z.device)
    with _Timed("patch_embed", out.numel() * 2) as tm:
        rc = _fn(lib, "vsb_patch_embed", z)(_p(z), _p(weight), _p(bias), _p(pos), _p(out), B, Cin, T, H, W, Cin * T * H * W,
                                            T * H * W, H * W, ph, pw, Cc, s0, s_local, st)
        if rc == 1:
            tm.cancel()
    if rc == 1:
        return None
    _lib.check(rc, "patch_embed")
    return out


def ln_modulate(x, mod, x_mask_u8, shift_row, scale_row, B, T, S, out=None, eps=1e-6, gamma=None, beta=None):
    """LayerNorm (optionally affine: gamma/beta) + modulate + per-frame select; x viewed as [B, T, S, C]."""
    lib, st = _prep(x, mod, x_mask_u8, out, gamma, beta)
    _bf16(x, "x")
    _same_dtype(x, mod, out, gamma, beta)
    Cc = x.shape[-1]
    out = torch.empty_like(x) if out is None else out
    with _Timed("ln_modulate", 2 * x.numel() * 2):
        if gamma is None and beta is None:  # STDiT3 / Latte: LayerNorm without affine parameters
            rc = _fn(lib, "vsb_ln_modulate", x)(_p(x), _p(out), _p(mod), _p(x_mask_u8), shift_row, scale_row, B, T, S, Cc, eps, st)
        else:  # CogVideoXLayerNormZero / norm_final / AdaLayerNorm: nn.LayerNorm with weight and bias in front
            rc = _fn(lib, "vsb_ln_modulate_affine", x)(_p(x), _p(out), _p(mod), _p(x_mask_u8), _p(gamma), _p(beta), shift_row,
                                                       scale_row, B, T, S, Cc, eps, st)
        _lib.check(rc, "ln_modulate")
    return out


def gate_residual(x, y, mod, x_mask_u8, gate_row, B, T, S, out=None, cache_out=None):
    lib, st = _prep(x, y, mod, x_mask_u8, out, cache_out)
    _same_dtype(x, y, mod, out, cache_out)
    Cc = x.shape[-1]
    out = torch.empty_like(x) if out is None else out
    with _Timed("gate_residual", (3 + (cache_out is not None)) * x.numel() * 2):
        _lib.check(
            _fn(lib, "vsb_gate_residual", x)(_p(x), _p(y), _p(out), _p(cache_out), _p(mod), _p(x_mask_u8), gate_row, B, T, S, Cc,
                                  st),
            "gate_residual",
        )
    return out


def residual_add(x, y, out=None):
    lib, st = _prep(x, y, out)
    _same_dtype(x, y, out)
    out = torch.empty_like(x) if out is None else out
    with _Timed("residual_add", 3 * x.numel() * 2):
        _lib.check(_fn(lib, "vsb_residual_add", x)(_p(x), _p(y), _p(out), x.numel(), st), "residual_add")
    return out


def dwconv_shuffle(x, w_taps, bias, B, T, H, W, ksize, down):
    """Depth-wise conv (kernel ksize = (kt, kh, kw), zero "same" padding) + bias + shortcut of x [B, T*H*W, C], stored in
    the sub-grid order [(B dt dh dw), (T/dt H/dh W/dw), C] of down = (dt, dh, dw); w_taps [kt*kh*kw, C] tap-major."""
    lib, st = _prep(x, w_taps, bias)
    _bf16(x, "x")
    _same_dtype(x, w_taps, bias)
    Cc = x.shape[-1]
    dt, dh, dw = down
    out = torch.empty(B * dt * dh * dw, (T // dt) * (H // dh) * (W // dw), Cc, dtype=x.dtype, device=x.device)
    with _Timed("dwconv_shuffle", 2 * x.numel() * 2):
        _lib.check(_fn(lib, "vsb_dwconv_shuffle", x)(_p(x), _p(w_taps), _p(bias), _p(out), B, T, H, W, Cc, *ksize, dt, dh, dw, st),
                   "dwconv_shuffle")
    return out


def gate_residual_unshuffle(x, y, mod, gate_row, B, T, H, W, down, out=None):
    """out = x + gate * y with y in the sub-grid order of dwconv_shuffle (read through the inverse regrouping)."""
    lib, st = _prep(x, y, mod, out)
    _same_dtype(x, y, mod, out)
    Cc = x.shape[-1]
    out = torch.empty_like(x) if out is None else out
    with _Timed("gate_residual", 3 * x.numel() * 2):
        _lib.check(_fn(lib, "vsb_gate_residual_unshuffle", x)(_p(x), _p(y), _p(out), _p(mod), gate_row, B, T, H, W, Cc, *down, st),
                   "gate_residual_unshuffle")
    return out


def dwconv_ffn(h, w_taps, bias, BT, H, W):
    """h + dw5x5(h) + dw3x3(h) + dw1x1(h) per frame of h [BT, H, W, C] (token-major); w_taps [35, C], bias [3, C]."""
    lib, st = _prep(h, w_taps, bias)
    _bf16(h, "h")
    _same_dtype(h, w_taps, bias)
    Cc = h.shape[-1]
    out = torch.empty_like(h)
    with _Timed("dwconv_ffn", 2 * h.numel() * 2):
        _lib.check(_fn(lib, "vsb_dwconv_ffn", h)(_p(h), _p(w_taps), _p(bias), _p(out), BT, H, W, Cc, st), "dwconv_ffn")
    return out


def kv_compress(x, w_taps, bias, ln_w, ln_b, B, T, H, W, window, pad_t=0, eps=1e-5, round_conv=True):
    """LayerNorm(depth-wise conv(x) + bias) with stride = window (kt, kh, kw) over x [B, T, H, W, C] (token-major), after
    pad_t leading copies of frame 0; returns [B, (T+pad_t)//kt, H//kh, W//kw, C].  w_taps [kt*kh*kw, C] tap-major.
    round_conv: round the conv before the bias is added (torch's cuDNN path) instead of once after it (ATen's native one)."""
    lib, st = _prep(x, w_taps, bias, ln_w, ln_b)
    _bf16(x, "x")
    _same_dtype(x, w_taps, bias, ln_w, ln_b)
    Cc = x.shape[-1]
    kt, kh, kw = window
    out = torch.empty(B, (T + pad_t) // kt, H // kh, W // kw, Cc, dtype=x.dtype, device=x.device)
    with _Timed("kv_compress", (x.numel() + out.numel()) * 2):
        _lib.check(_fn(lib, "vsb_kv_compress", x)(_p(x), _p(w_taps), _p(bias), _p(ln_w), _p(ln_b), _p(out), B, T, H, W, Cc, kt, kh,
                                                  kw, pad_t, eps, int(bool(round_conv)), st), "kv_compress")
    return out


VAE_GN_CHUNKS = 256  # VSB_GN_CHUNKS of include/vsb200.h


def vae_conv3d(x, w_packed, bias, cout, kt, resid=None, round_conv=True):
    """Causal (kt, 3, 3) convolution of x [B, kt-1+T, H, W, Cin] (causal context first, channels-last) with zero spatial
    padding; w_packed [Cout_pad, kt*9, Cin_pad] tap-major (pack_conv_weight); returns [B, T, H, W, cout] = conv + bias
    [+ resid].  round_conv: round the convolution before the bias is added (torch's cuDNN path)."""
    lib, st = _prep(x, w_packed, bias, resid)
    _bf16(x, "x")
    _same_dtype(x, w_packed, bias, resid)
    B, Tin, H, W, Cin = x.shape
    T = Tin - (kt - 1)
    out = torch.empty(B, T, H, W, cout, dtype=x.dtype, device=x.device)
    with _Timed("vae_conv3d", 2 * B * T * H * W * cout * Cin * kt * 9):
        _lib.check(_fn(lib, "vsb_vae_conv3d", x)(_p(x), _p(w_packed), _p(bias), _p(resid), _p(out), B, T, H, W, Cin, cout, kt,
                                                 int(bool(round_conv)), st), "vae_conv3d")
    return out


def vae_conv_time(x, w_packed, bias, cout, kt, resid=None, mix=None, round_conv=True):
    """(kt, 1, 1) convolution of x [B, kt-1+T, H, W, Cin] (channels-last, the time padding materialised as frames of x);
    w_packed [Cout, kt, Cin] (pack_conv_weight of a [Cout, Cin, kt, 1, 1] weight); returns [B, T, H, W, cout] = conv +
    bias [+ resid].  mix = (a, b): instead out = a * resid + b * (resid + conv + bias), each op rounded (the SVD
    temporal decoder's TemporalResnetBlock sum and AlphaBlender)."""
    lib, st = _prep(x, w_packed, bias, resid)
    _bf16(x, "x")
    _same_dtype(x, w_packed, bias, resid)
    B, Tin, H, W, Cin = x.shape
    T = Tin - (kt - 1)
    if mix is not None and resid is None:
        raise _lib.VsbError("vae_conv_time: mix needs resid")
    a, b = (0.0, 0.0) if mix is None else (float(mix[0]), float(mix[1]))
    out = torch.empty(B, T, H, W, cout, dtype=x.dtype, device=x.device)
    with _Timed("vae_conv_time", 2 * B * T * H * W * cout * Cin * kt):
        _lib.check(_fn(lib, "vsb_vae_conv_time", x)(_p(x), _p(w_packed), _p(bias), _p(resid), _p(out), B, T, H, W, Cin, cout, kt,
                                                    int(mix is not None), a, b, int(bool(round_conv)), st), "vae_conv_time")
    return out


def vae_conv_down(x, w_packed, bias, cout, kt, round_conv=True):
    """The OpenSora v1.2 VAE encoder's down-sampling convolutions of x [B, Tin, Hin, Win, Cin] (channels-last), w_packed
    as for vae_conv3d; returns conv + bias.  kt = 1: Downsample2D (zero pad right and bottom by 1, 3x3 conv, stride 2 in
    H and W) -> [B, Tin, (Hin - 2) // 2 + 1, (Win - 2) // 2 + 1, cout].  kt = 3: the causal (3, 3, 3) conv with stride
    (2, 1, 1) and one zero frame in front (not materialised) -> [B, (Tin - 2) // 2 + 1, Hin, Win, cout]."""
    lib, st = _prep(x, w_packed, bias)
    _bf16(x, "x")
    _same_dtype(x, w_packed, bias)
    B, Tin, Hin, Win, Cin = x.shape
    if kt == 1:
        stride_t, stride_hw, T, H, W = 1, 2, Tin, (Hin - 2) // 2 + 1, (Win - 2) // 2 + 1
    elif kt == 3:
        stride_t, stride_hw, T, H, W = 2, 1, (Tin - 2) // 2 + 1, Hin, Win
    else:
        raise _lib.VsbError(f"vae_conv_down: kt={kt} (need 1: spatial stride 2, or 3: temporal stride 2)")
    out = torch.empty(B, max(T, 1), max(H, 1), max(W, 1), cout, dtype=x.dtype, device=x.device)
    with _Timed("vae_conv_down", 2 * out.numel() * Cin * kt * 9):
        _lib.check(_fn(lib, "vsb_vae_conv_down", x)(_p(x), _p(w_packed), _p(bias), _p(out), B, Tin, Hin, Win, Cin, cout, kt,
                                                    stride_t, stride_hw, int(bool(round_conv)), st), "vae_conv_down")
    return out


def vae_time_conv_rgb(x, weight, bias):
    """Conv3d 3 -> 3, kernel (3, 1, 1), padding (1, 0, 0), + bias, of x [B, T, H, W, 3]; weight [3, 3, 3, 1, 1] as stored."""
    lib, st = _prep(x, weight, bias)
    _bf16(x, "x")
    _same_dtype(x, weight, bias)
    B, T, H, W, Cc = x.shape
    if Cc != 3 or tuple(weight.shape) != (3, 3, 3, 1, 1):
        raise _lib.VsbError("vae_time_conv_rgb: needs 3 channels and a [3, 3, 3, 1, 1] weight")
    out = torch.empty_like(x)
    with _Timed("vae_time_conv_rgb", 2 * x.numel() * 2):
        _lib.check(_fn(lib, "vsb_vae_time_conv_rgb", x)(_p(x), _p(weight), _p(bias), _p(out), B, T, H, W, st), "vae_time_conv_rgb")
    return out


def pack_conv_weight(w):
    """[Cout, Cin, (kt,) 3, 3] conv weight -> [Cout_pad, kt*9, Cin_pad] tap-major, Cout and Cin zero padded to multiples
    of 64 (include/vsb200.h); a (kt, 1, 1) weight [Cout, Cin, kt, 1, 1] -> [Cout_pad, kt, Cin_pad] likewise."""
    if w.dim() == 4:
        w = w[:, :, None]
    cout, cin, kt = w.shape[0], w.shape[1], w.shape[2]
    taps = kt * w.shape[3] * w.shape[4]
    cout_pad, cin_pad = -(-cout // 64) * 64, -(-cin // 64) * 64
    p = torch.zeros(cout_pad, taps, cin_pad, dtype=w.dtype, device=w.device)
    p[:cout, :, :cin] = w.permute(0, 2, 3, 4, 1).reshape(cout, taps, cin)
    return p


def vae_groupnorm_stats(x, groups, eps):
    """fp32 [B, groups, 2] (mean, rstd) of nn.GroupNorm over x [B, T, H, W, C] (channels-last)."""
    lib, st = _prep(x)
    _bf16(x, "x")
    B, C = x.shape[0], x.shape[-1]
    P = x.numel() // (B * C)
    stats = torch.empty(B, groups, 2, dtype=torch.float32, device=x.device)
    ws = torch.empty(B * VAE_GN_CHUNKS * C * 2, dtype=torch.float32, device=x.device)
    with _Timed("vae_groupnorm_stats", x.numel() * 2):
        _lib.check(_fn(lib, "vsb_vae_groupnorm_stats", x)(_p(x), _p(stats), _p(ws), B, P, C, groups, float(eps), st),
                   "vae_groupnorm_stats")
    return stats


def vae_spatial_norm_silu(f, stats, gamma, beta, zyb, out, t_off=0):
    """silu(GroupNorm(f) * zy + zb) of f [B, T, H, W, C] into frames t_off .. t_off+T-1 of out [B, T_out, H, W, C]; zyb
    [B, Tz, h, w, 2C] = conv_y | conv_b of the latent, gathered with F.interpolate's nearest rule; stats from
    vae_groupnorm_stats."""
    lib, st = _prep(f, stats, gamma, beta, zyb, out)
    _bf16(f, "f")
    _same_dtype(f, gamma, beta, zyb, out)
    B, T, H, W, C = f.shape
    _, Tz, h, w, _ = zyb.shape
    G = stats.shape[1]
    with _Timed("vae_spatial_norm_silu", (2 * f.numel() + zyb.numel()) * 2):
        _lib.check(_fn(lib, "vsb_vae_spatial_norm_silu", f)(_p(f), _p(stats), _p(gamma), _p(beta), _p(zyb), _p(out), B, T, H, W, C,
                                                            G, Tz, h, w, t_off, out.shape[1], st), "vae_spatial_norm_silu")
    return out


def vae_upsample2x(x, compress_time):
    """Nearest 2x of x [B, T, H, W, C] in H and W, and in T when compress_time (first frame kept single for odd T)."""
    lib, st = _prep(x)
    _bf16(x, "x")
    B, T, H, W, C = x.shape
    T2 = (2 * T - (T % 2)) if (compress_time and T > 1) else T
    out = torch.empty(B, T2, 2 * H, 2 * W, C, dtype=x.dtype, device=x.device)
    with _Timed("vae_upsample2x", (x.numel() + out.numel()) * 2):
        _lib.check(_fn(lib, "vsb_vae_upsample2x", x)(_p(x), _p(out), B, T, H, W, C, int(bool(compress_time)), st), "vae_upsample2x")
    return out


def vae_groupnorm_act(x, stats, gamma, beta, out=None, t_off=0, act=True):
    """GroupNorm of x [B, T, H, W, C] with stats from vae_groupnorm_stats, then x * sigmoid(x) when act is true (1),
    F.silu (one rounding) when act == 2, into frames t_off .. t_off+T-1 of out [B, T_out, H, W, C] (default: a new
    [B, T, H, W, C])."""
    lib, st = _prep(x, stats, gamma, beta, out)
    _bf16(x, "x")
    _same_dtype(x, gamma, beta, out)
    B, T, H, W, C = x.shape
    out = torch.empty_like(x) if out is None else out
    with _Timed("vae_groupnorm_act", 2 * x.numel() * 2):
        _lib.check(_fn(lib, "vsb_vae_groupnorm_act", x)(_p(x), _p(stats), _p(gamma), _p(beta), _p(out), B, T, H, W, C, stats.shape[1],
                                                        t_off, out.shape[1], 2 if act == 2 else int(bool(act)), st), "vae_groupnorm_act")
    return out


def vae_depth_to_time(x, out=None, t_off=0):
    """rearrange "B (C ts) T H W -> B C (T ts) H W" (ts = 2) of x [B, T, H, W, 2C] into frames t_off .. t_off+2T-1 of out
    [B, T_out, H, W, C] (default: a new [B, 2T, H, W, C])."""
    lib, st = _prep(x, out)
    _bf16(x, "x")
    _same_dtype(x, out)
    B, T, H, W, C2 = x.shape
    if C2 % 2:
        raise _lib.VsbError(f"vae_depth_to_time: odd channel count {C2}")
    out = torch.empty(B, 2 * T, H, W, C2 // 2, dtype=x.dtype, device=x.device) if out is None else out
    with _Timed("vae_depth_to_time", 2 * x.numel() * 2):
        _lib.check(_fn(lib, "vsb_vae_depth_to_time", x)(_p(x), _p(out), B, T, H, W, C2 // 2, t_off, out.shape[1], st),
                   "vae_depth_to_time")
    return out


def vae_upsample_linear2x(x, spatial, temporal, out=None, t_off=0):
    """Trilinear (align_corners=False) 2x of x [B, T, H, W, C] in H and W (spatial) and in T over frames 1.. (temporal),
    into frames t_off.. of out [B, T_out, Ho, Wo, C] (default: a new tensor of exactly the output frames)."""
    lib, st = _prep(x, out)
    _bf16(x, "x")
    _same_dtype(x, out)
    B, T, H, W, C = x.shape
    To = 2 * T - 1 if (temporal and T > 1) else T
    if out is None:
        out = torch.empty(B, To, H * (2 if spatial else 1), W * (2 if spatial else 1), C, dtype=x.dtype, device=x.device)
    with _Timed("vae_upsample_linear2x", (x.numel() + out.numel()) * 2):
        _lib.check(_fn(lib, "vsb_vae_upsample_linear2x", x)(_p(x), _p(out), B, T, H, W, C, int(bool(spatial)), int(bool(temporal)),
                                                            t_off, out.shape[1], st), "vae_upsample_linear2x")
    return out


def vae_mix(xbuf, y, alpha, one_minus_alpha, t_off=0):
    """alpha * x + one_minus_alpha * y, each op rounded, x = frames t_off.. of xbuf [B, T_x, H, W, C], y [B, T, H, W, C]."""
    lib, st = _prep(xbuf, y)
    _same_dtype(xbuf, y)
    B, T = y.shape[0], y.shape[1]
    out = torch.empty_like(y)
    with _Timed("vae_mix", 3 * y.numel() * 2):
        _lib.check(_fn(lib, "vsb_vae_mix", y)(_p(xbuf), _p(y), _p(out), B, T, y[0, 0].numel(), t_off, xbuf.shape[1], float(alpha),
                                              float(one_minus_alpha), st), "vae_mix")
    return out


def vae_attn_split(qkv, C, mixed):
    """qkv [B, T, H, W, 3C] -> per-frame q [B*T, P, C], k [B*T, Pp, C], vt [B*T, C, Pp] (P = H*W, Pp = P rounded up to 8,
    zero past P); mixed: AttnBlock3D's frame / channel mixing."""
    lib, st = _prep(qkv)
    _bf16(qkv, "qkv")
    B, T = qkv.shape[0], qkv.shape[1]
    P = qkv[0, 0].numel() // (3 * C)
    Pp = -(-P // 8) * 8
    q = torch.empty(B * T, P, C, dtype=qkv.dtype, device=qkv.device)
    k = torch.empty(B * T, Pp, C, dtype=qkv.dtype, device=qkv.device)
    vt = torch.empty(B * T, C, Pp, dtype=qkv.dtype, device=qkv.device)
    with _Timed("vae_attn_split", 2 * qkv.numel() * 2):
        _lib.check(_fn(lib, "vsb_vae_attn_split", qkv)(_p(qkv), _p(q), _p(k), _p(vt), B, T, P, Pp, C, int(bool(mixed)), st),
                   "vae_attn_split")
    return q, k, vt


def vae_attn_softmax_(S, P, scale):
    """In place: softmax over the first P columns of bf16(S * scale), S [rows, Pp]; columns P.. become zero."""
    lib, st = _prep(S)
    _bf16(S, "S")
    rows, Pp = S.numel() // S.shape[-1], S.shape[-1]
    with _Timed("vae_attn_softmax", 2 * S.numel() * 2):
        _lib.check(_fn(lib, "vsb_vae_attn_softmax", S)(_p(S), rows, P, Pp, float(scale), st), "vae_attn_softmax")
    return S


def vae_attn_merge(o, B, T, H, W):
    """AttnBlock3D's output scatter: o [B*T, P, C] (pseudo-frames) -> [B, T, H, W, C]."""
    lib, st = _prep(o)
    _bf16(o, "o")
    C = o.shape[-1]
    out = torch.empty(B, T, H, W, C, dtype=o.dtype, device=o.device)
    with _Timed("vae_attn_merge", 2 * o.numel() * 2):
        _lib.check(_fn(lib, "vsb_vae_attn_merge", o)(_p(o), _p(out), B, T, H * W, C, st), "vae_attn_merge")
    return out


def qk_rmsnorm_(qkv, wq, wk, H, D, eps=1e-6, rope_cos=None, rope_sin=None, pos_div=1, pos_mod=1):
    """In-place per-head RMSNorm of q and k; with rope tables also RoPE at position (row // pos_div) % pos_mod."""
    lib, st = _prep(qkv, wq, wk, rope_cos, rope_sin)
    rows = qkv.numel() // (3 * H * D)
    with _Timed("qk_rmsnorm", 4 * rows * H * D * 2):
        _lib.check(_fn(lib, "vsb_qk_rmsnorm_rope", qkv)(_p(qkv), _p(wq), _p(wk), rows, H, D, eps, _p(rope_cos), _p(rope_sin),
                                           int(pos_div), int(pos_mod), st), "qk_rmsnorm")
    return qkv


def qk_rope_halves_(qkv, rope_cos, rope_sin_signed, H, D, half, pos_div=1, pos_mod=1):
    """In-place half-rotation RoPE of q and k (Open-Sora-Plan RoPE1D / 2D / 3D): tables [pos_mod, D] fp32, the sign of
    rotate_half folded into the sin table; token row r uses table row (r // pos_div) % pos_mod."""
    lib, st = _prep(qkv, rope_cos, rope_sin_signed)
    rows = qkv.numel() // (3 * H * D)
    with _Timed("qk_rmsnorm", 4 * rows * H * D * 2):
        _lib.check(_fn(lib, "vsb_qk_rope_halves", qkv)(_p(qkv), rows, H, D, int(half), _p(rope_cos), _p(rope_sin_signed),
                                                       int(pos_div), int(pos_mod), st), "qk_rope_halves")
    return qkv


def qk_layernorm_(qkv, wq, bq, wk, bk, H, D, eps=1e-6):
    lib, st = _prep(qkv, wq, bq, wk, bk)
    rows = qkv.numel() // (3 * H * D)
    with _Timed("qk_rmsnorm", 4 * rows * H * D * 2):
        _lib.check(_fn(lib, "vsb_qk_layernorm", qkv)(_p(qkv), _p(wq), _p(bq), _p(wk), _p(bk), rows, H, D, eps, st), "qk_layernorm")
    return qkv


def attn_short(qkv, wq, wk, rope_cos, rope_sin, n_outer, n_inner, outer_stride, inner_stride, tok_stride, n, H, D,
               scale, out=None, eps=1e-6, flags: int = 0):
    lib, st = _prep(qkv, wq, wk, rope_cos, rope_sin, out)
    rows = qkv.numel() // (3 * H * D)
    out = torch.empty(rows, H * D, dtype=qkv.dtype, device=qkv.device) if out is None else out
    with _Timed("attn_short", 4 * rows * H * D * 2):
        _lib.check(
            _fn(lib, "vsb_attn_short", qkv)(_p(qkv), _p(out), _p(wq), _p(wk), _p(rope_cos), _p(rope_sin), n_outer, n_inner,
                               outer_stride, inner_stride, tok_stride, n, H, D, eps, scale, flags, st),
            "attn_short",
        )
    return out


def gemm_bias_act(a, w, bias=None, act: int = 0, out=None):
    """out[..., N] = act(a[..., K] @ w[N, K]^T + bias)."""
    lib, st = _prep(a, w, bias, out)
    _bf16(a, "a"), _bf16(w, "w"), _bf16(bias, "bias")
    K = a.shape[-1]
    M = a.numel() // K
    N = w.shape[0]
    if w.shape[1] != K:
        raise _lib.VsbError("gemm: K mismatch")
    _same_dtype(a, w, bias, out)
    out = torch.empty(*a.shape[:-1], N, dtype=a.dtype, device=a.device) if out is None else out
    with _Timed("gemm", 2 * M * N * K):
        _lib.check(_fn(lib, "vsb_gemm_bias_act", a)(_p(a), _p(w), _p(bias), _p(out), M, N, K, act, st), "gemm_bias_act")
    return out


def gemm_bias_residual(a, w, bias, resid, mod=None, x_mask_u8=None, gate_row: int = -1, B=1, T=1, S=1, out=None):
    """out = resid + [gate *] (a @ w^T + bias) with the branch fused into the GEMM epilogue (out defaults to resid)."""
    lib, st = _prep(a, w, bias, resid, mod, x_mask_u8, out)
    K = a.shape[-1]
    M = a.numel() // K
    N = w.shape[0]
    out = resid if out is None else out
    with _Timed("gemm", 2 * M * N * K):
        _lib.check(_fn(lib, "vsb_gemm_bias_residual", a)(_p(a), _p(w), _p(bias), _p(resid), _p(out), _p(mod), _p(x_mask_u8),
                                                       gate_row, M, N, K, B, T, S, st), "gemm_bias_residual")
    return out


def gemm_kernel_name(M: int, N: int, K: int, act: int = 0, residual: bool = False) -> str:
    """The kernel instance gemm_bias_act (act) or gemm_bias_residual (residual=True) launches for an M x N x K GEMM."""
    lib = _lib.load()
    name = lib.vsb_gemm_kernel_name(M, N, K, act, int(residual)).decode()
    if not name:
        raise _lib.VsbError(f"gemm_kernel_name: bad arguments M={M} N={N} K={K} act={act} residual={residual}")
    return name


def _fp8_codes(t, name):
    if t.dtype not in (torch.float8_e4m3fn, torch.uint8):
        raise _lib.VsbError(f"{name} must hold e4m3 codes (float8_e4m3fn or uint8), got {t.dtype}")


def quant_rows_fp8(x):
    """(q, scale): e4m3 codes [..., K] (float8_e4m3fn) and fp32 per-row scales [...] of x [..., K], by the rule of
    include/vsb200.h (scale = amax / 448 of the row, 1 for an all-zero row)."""
    lib, st = _prep(x)
    _bf16(x, "x")
    K = x.shape[-1]
    M = x.numel() // K
    q = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device=x.device)
    scale = torch.empty(x.shape[:-1], dtype=torch.float32, device=x.device)
    with _Timed("quant", 3 * M * K + 4 * M):
        _lib.check(_fn(lib, "vsb_quant_rows_fp8", x)(_p(x), _p(q), _p(scale), M, K, st), "quant_rows_fp8")
    return q, scale


def ln_modulate_fp8(x, mod, x_mask_u8, shift_row, scale_row, B, T, S, eps=1e-6):
    """ln_modulate with its output quantized: (q, scale) == quant_rows_fp8(ln_modulate(...)) bit for bit."""
    lib, st = _prep(x, mod, x_mask_u8)
    _bf16(x, "x")
    _same_dtype(x, mod)
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    q = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device=x.device)
    scale = torch.empty(x.shape[:-1], dtype=torch.float32, device=x.device)
    with _Timed("ln_modulate", 3 * x.numel() + 4 * rows):
        _lib.check(_fn(lib, "vsb_ln_modulate_fp8", x)(_p(x), _p(q), _p(scale), _p(mod), _p(x_mask_u8), shift_row, scale_row, B, T,
                                                      S, Cc, eps, st), "ln_modulate_fp8")
    return q, scale


def gemm_fp8_bias_act(a, a_scale, w, w_scale, bias=None, act: int = 0, out=None, dtype=torch.bfloat16):
    """out[..., N] = act(bf16(acc * a_scale[m] * w_scale[n] + bias)) with a [..., K], w [N, K] e4m3 codes; out in bias's
    16-bit dtype (else dtype)."""
    lib, st = _prep(a, a_scale, w, w_scale, bias, out)
    _fp8_codes(a, "a"), _fp8_codes(w, "w"), _bf16(bias, "bias")
    K = a.shape[-1]
    M = a.numel() // K
    N = w.shape[0]
    if w.shape[1] != K:
        raise _lib.VsbError("gemm_fp8: K mismatch")
    ref = bias if bias is not None else (out if out is not None else torch.empty(0, dtype=dtype))
    _same_dtype(bias, out)
    out = torch.empty(*a.shape[:-1], N, dtype=ref.dtype, device=a.device) if out is None else out
    with _Timed("gemm_fp8", 2 * M * N * K):
        _lib.check(_fn(lib, "vsb_gemm_fp8_bias_act", ref)(_p(a), _p(a_scale), _p(w), _p(w_scale), _p(bias), _p(out), M, N, K, act,
                                                          st), "gemm_fp8_bias_act")
    return out


def gemm_fp8_bias_residual(a, a_scale, w, w_scale, bias, resid, mod=None, x_mask_u8=None, gate_row: int = -1, B=1, T=1, S=1,
                           out=None):
    """out = resid + [gate *] bf16(acc * a_scale * w_scale + bias), fused as gemm_bias_residual (out defaults to resid)."""
    lib, st = _prep(a, a_scale, w, w_scale, bias, resid, mod, x_mask_u8, out)
    _fp8_codes(a, "a"), _fp8_codes(w, "w"), _bf16(resid, "resid")
    _same_dtype(bias, resid, mod, out)
    K = a.shape[-1]
    M = a.numel() // K
    N = w.shape[0]
    out = resid if out is None else out
    with _Timed("gemm_fp8", 2 * M * N * K):
        _lib.check(_fn(lib, "vsb_gemm_fp8_bias_residual", resid)(_p(a), _p(a_scale), _p(w), _p(w_scale), _p(bias), _p(resid), _p(out),
                                                                 _p(mod), _p(x_mask_u8), gate_row, M, N, K, B, T, S, st),
                   "gemm_fp8_bias_residual")
    return out


def gemm_fp8_kernel_name(M: int, N: int, K: int, act: int = 0, residual: bool = False) -> str:
    """The kernel instance gemm_fp8_bias_act (act) or gemm_fp8_bias_residual (residual=True) launches."""
    name = _lib.load().vsb_gemm_fp8_kernel_name(M, N, K, act, int(residual)).decode()
    if not name:
        raise _lib.VsbError(f"gemm_fp8_kernel_name: bad arguments M={M} N={N} K={K} act={act} residual={residual}")
    return name


def attn_flash(q, k, v, nb, nq, nk, H, D, q_row_stride, q_batch_stride, kv_row_stride, kv_batch_stride, scale,
               kv_lens: Optional[Sequence[int]] = None, out=None, out_row_stride=None, out_batch_stride=None):
    """q/k/v: tensors whose data_ptr() is the first element of the strided view (may be slices of one buffer).
    out_row_stride / out_batch_stride (elements): strided output view starting at out.data_ptr() (default: contiguous
    [nb, nq, H*D])."""
    lib = _lib.load()
    if not q.is_cuda:
        raise _lib.VsbError("vsb200 kernels need CUDA tensors (no CPU fallback)")
    _init_dev(lib, q.device.index)
    st = torch.cuda.current_stream().cuda_stream
    _same_dtype(q, k, v, out)
    out = torch.empty(nb, nq, H * D, dtype=q.dtype, device=q.device) if out is None else out
    lens = None
    if kv_lens is not None:
        lens = (C.c_int * len(kv_lens))(*[int(v_) for v_ in kv_lens])
    with _Timed("attn_flash", 4 * nb * H * nq * nk * D):
        _lib.check(
            _fn(lib, "vsb_attn_flash_strided", q)(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), nb, nq, nk, H, D,
                                       q_row_stride, q_batch_stride, kv_row_stride, kv_batch_stride,
                                       H * D if out_row_stride is None else out_row_stride,
                                       nq * H * D if out_batch_stride is None else out_batch_stride, lens, scale, st),
            "attn_flash",
        )
    return out


def pab_gate(on: bool, timestep: Optional[int], count: int, rng: int, lo: int, hi: int, steps: int):
    lib = _lib.load()
    c = C.c_int(count)
    rc = lib.vsb_pab_gate(int(bool(on)), int(timestep is not None), int(timestep or 0), C.byref(c), int(rng or 1),
                          int(lo), int(hi), int(steps))
    _lib.check(rc, "pab_gate")
    return bool(rc), c.value
