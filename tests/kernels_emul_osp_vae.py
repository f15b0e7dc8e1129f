"""TEST INFRASTRUCTURE ONLY -- torch stand-ins for the Open-Sora-Plan VAE decoder entries of ``videosys_b200.kernels``, on
top of the stand-ins of tests/kernels_emul_vae.py.  Each takes exactly the arguments of the function it replaces, with the
kernels' channels-last layouts, and computes what the reference's eager chain computes (F.group_norm, x * torch.sigmoid(x),
F.interpolate trilinear, torch.bmm, softmax, the reshapes of AttnBlock3D), on whatever device and dtype the tensors have:
in fp32 on the CPU it is the host logic's check against the reference, in 16 bits on the GPU it is the eager 16-bit
decoder the kernels are measured against.  The product never imports this file."""
import torch
import torch.nn.functional as F

from tests import kernels_emul_vae as EV
from videosys_b200 import kernels


def vae_groupnorm_act(x, stats, gamma, beta, out=None, t_off=0, act=True):
    B, T, H, W, C = x.shape
    G = stats.shape[1]
    # F.group_norm on the GPU with the given statistics: mean and rstd kept in the input dtype, a = rstd * gamma,
    # b = -a * mean + beta, y = a * x + b in fp32
    mean = stats[..., 0].to(x.dtype).float().repeat_interleave(C // G, 1).view(B, 1, 1, 1, C)
    rstd = stats[..., 1].to(x.dtype).float().repeat_interleave(C // G, 1).view(B, 1, 1, 1, C)
    a = rstd * gamma.float()
    n = (a * x.float() + (beta.float() - a * mean)).to(x.dtype)
    y = n * torch.sigmoid(n) if act else n
    if out is None:
        return y.contiguous()
    out[:, t_off:t_off + T] = y
    return out


def vae_upsample_linear2x(x, spatial, temporal, out=None, t_off=0):
    s = 2 if spatial else 1
    xi = x.permute(0, 4, 1, 2, 3)
    if temporal and xi.shape[2] > 1:
        first = F.interpolate(xi[:, :, :1], scale_factor=(1, s, s), mode="trilinear")
        rest = F.interpolate(xi[:, :, 1:], scale_factor=(2, s, s), mode="trilinear")
        y = torch.cat([first, rest], dim=2)
    else:
        y = F.interpolate(xi, scale_factor=(1, s, s), mode="trilinear")
    y = y.permute(0, 2, 3, 4, 1)
    if out is None:
        return y.contiguous()
    out[:, t_off:t_off + y.shape[1]] = y
    return out


def vae_mix(xbuf, y, alpha, one_minus_alpha, t_off=0):
    x = xbuf[:, t_off:t_off + y.shape[1]]
    a = torch.tensor([alpha], dtype=y.dtype, device=y.device)
    oma = torch.tensor([one_minus_alpha], dtype=y.dtype, device=y.device)
    return (a * x + oma * y).contiguous()


def _to_reference_frames(t, mixed):
    """[B, T, H, W, C] -> the reference's (b*t, c, h*w): AttnBlock3D reshapes b c t h w directly, the Fix permutes first."""
    B, T, H, W, C = t.shape
    x = t.permute(0, 4, 1, 2, 3)
    if not mixed:
        x = x.permute(0, 2, 1, 3, 4)
    return x.reshape(B * T, C, H * W)


def vae_attn_split(qkv, C, mixed):
    B, T, H, W, _ = qkv.shape
    P = H * W
    Pp = -(-P // 8) * 8
    q, k, v = (_to_reference_frames(qkv[..., i * C:(i + 1) * C], mixed) for i in range(3))
    kp = torch.zeros(B * T, Pp, C, dtype=qkv.dtype, device=qkv.device)
    vt = torch.zeros(B * T, C, Pp, dtype=qkv.dtype, device=qkv.device)
    kp[:, :P] = k.transpose(1, 2)
    vt[:, :, :P] = v
    return q.transpose(1, 2).contiguous(), kp, vt


def vae_attn_softmax_(S, P, scale):
    S[..., :P] = F.softmax(S[..., :P] * scale, dim=-1)
    S[..., P:] = 0
    return S


def vae_attn_merge(o, B, T, H, W):
    C = o.shape[-1]
    return o.transpose(1, 2).reshape(B, C, T, H, W).permute(0, 2, 3, 4, 1).contiguous()


NAMES = ["vae_groupnorm_act", "vae_upsample_linear2x", "vae_mix", "vae_attn_split", "vae_attn_softmax_", "vae_attn_merge"]


def emulate(monkeypatch):
    """tests/kernels_emul_vae.emulate plus the Open-Sora-Plan VAE stand-ins, for the duration of one test."""
    EV.emulate(monkeypatch)
    for n in NAMES:
        monkeypatch.setattr(kernels, n, globals()[n])
