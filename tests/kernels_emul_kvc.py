"""TEST INFRASTRUCTURE ONLY -- torch/CPU stand-in for ``kv_compress`` (Open-Sora-Plan v1.1.0's KV compression), on top of the
stand-ins of tests/kernels_emul.py.  Same conventions: it takes exactly the arguments of the function it replaces; the
product never imports this file."""
import torch
import torch.nn.functional as F

from tests import kernels_emul as E
from videosys_b200 import kernels


def kv_compress(x, w_taps, bias, ln_w, ln_b, B, T, H, W, window, pad_t=0, eps=1e-5, round_conv=True):
    """The reference's eager chain (open_sora_plan_v110_transformer_3d.py:1181-1197): depth-wise conv with stride = window
    over the channels-first view, + bias, LayerNorm over C; returns [B, T', H', W', C] token-major."""
    C = x.shape[-1]
    kt, kh, kw = window
    v = x.reshape(B, T, H, W, C)
    if pad_t:
        v = torch.cat([v[:, :1].expand(B, pad_t, H, W, C), v], 1)
    xi = v.permute(0, 4, 1, 2, 3)  # [B, C, T, H, W]
    y = F.conv3d(xi, w_taps.t().reshape(C, 1, kt, kh, kw), bias, stride=window, groups=C)
    y = y.permute(0, 2, 3, 4, 1)
    return F.layer_norm(y, (C,), ln_w, ln_b, eps).contiguous()


def emulate(monkeypatch):
    """tests/kernels_emul.emulate plus the KV-compression stand-in, for the duration of one test."""
    E.emulate(monkeypatch)
    monkeypatch.setattr(kernels, "kv_compress", kv_compress)


def emulate_global():
    """The same for a spawned worker process."""
    E.emulate_global()
    kernels.kv_compress = kv_compress
