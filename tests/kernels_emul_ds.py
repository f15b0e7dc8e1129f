"""TEST INFRASTRUCTURE ONLY -- torch/CPU stand-ins for the kernels of Open-Sora-Plan v1.2.0's conv down-sampler path
(``dwconv_shuffle``, ``gate_residual_unshuffle``, ``dwconv_ffn`` and the erf-GELU epilogue ``gemm_bias_act(act=2)``), on top of
the stand-ins of tests/kernels_emul.py.  Same conventions: each takes exactly the arguments of the function it replaces;
the product never imports this file."""
import torch.nn.functional as F

from tests import kernels_emul as E
from videosys_b200 import kernels


def gemm_bias_act(a, w, bias=None, act=0, out=None):
    if act != 2:
        return E.gemm_bias_act(a, w, bias, act, out)
    y = F.gelu(F.linear(a, w, bias))
    if out is None:
        return y
    out.copy_(y.view(out.shape))
    return out


def _dw_weight(w_taps, C, k):
    return w_taps.t().reshape(C, 1, *k)


def dwconv_shuffle(x, w_taps, bias, B, T, H, W, ksize, down):
    C = x.shape[-1]
    kt, kh, kw = ksize
    dt, dh, dw = down
    v = x.reshape(B, T, H, W, C)
    if kt == 1:  # DownSampler2d: Conv2d per frame
        xi = v.reshape(B * T, H, W, C).permute(0, 3, 1, 2)
        y = F.conv2d(xi, _dw_weight(w_taps, C, (kh, kw)), bias.reshape(C), padding=(kh // 2, kw // 2), groups=C) + xi
        y = y.reshape(B, T, C, H, W).permute(0, 2, 1, 3, 4)
    else:
        xi = v.permute(0, 4, 1, 2, 3)
        y = F.conv3d(xi, _dw_weight(w_taps, C, ksize), bias.reshape(C), padding=(kt // 2, kh // 2, kw // 2), groups=C) + xi
    y = y.reshape(B, C, T // dt, dt, H // dh, dh, W // dw, dw)  # b d (t dt) (h dh) (w dw) -> (b dt dh dw) (t h w) d
    return y.permute(0, 3, 5, 7, 2, 4, 6, 1).reshape(B * dt * dh * dw, -1, C).contiguous()


def unshuffle(y, B, T, H, W, down):
    """[(b dt dh dw), (t h w), C] -> [b, (t dt h dh w dw), C]: DownSampler3d.reverse."""
    dt, dh, dw = down
    C = y.shape[-1]
    v = y.reshape(B, dt, dh, dw, T // dt, H // dh, W // dw, C)
    return v.permute(0, 4, 1, 5, 2, 6, 3, 7).reshape(B, T * H * W, C)


def gate_residual_unshuffle(x, y, mod, gate_row, B, T, H, W, down, out=None):
    return E.gate_residual(x, unshuffle(y, B, T, H, W, down), mod, None, gate_row, B, 1, T * H * W, out=out)


def dwconv_ffn(h, w_taps, bias, BT, H, W):
    C = h.shape[-1]
    xi = h.reshape(BT, H, W, C).permute(0, 3, 1, 2)
    out, o = xi, 0
    for i, k in enumerate((5, 3, 1)):
        out = out + F.conv2d(xi, _dw_weight(w_taps[o:o + k * k], C, (k, k)), bias[i], padding=k // 2, groups=C)
        o += k * k
    return out.permute(0, 2, 3, 1).reshape(h.shape).contiguous()


NAMES = ["gemm_bias_act", "dwconv_shuffle", "gate_residual_unshuffle", "dwconv_ffn"]


def emulate(monkeypatch):
    """tests/kernels_emul.emulate plus the down-sampler stand-ins, for the duration of one test."""
    E.emulate(monkeypatch)
    g = globals()
    for n in NAMES:
        monkeypatch.setattr(kernels, n, g[n])
