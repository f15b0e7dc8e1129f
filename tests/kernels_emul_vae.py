"""TEST INFRASTRUCTURE ONLY -- torch stand-ins for the VAE decoder entries of ``videosys_b200.kernels`` (the CogVideoX,
Open-Sora-Plan and OpenSora v1.2 decoders), on top of the stand-ins of tests/kernels_emul.py.  Each takes exactly the
arguments of the function it replaces, with the kernels' channels-last layouts, and computes what the reference's eager
chain computes (F.pad + F.conv3d on NCDHW, F.group_norm, x * torch.sigmoid(x) or F.silu, F.interpolate nearest and
trilinear, torch.bmm / softmax on the reshapes of AttnBlock3D, the einops rearrange of depth-to-time), on whatever device
and dtype the tensors have: in fp32 on the CPU it is the host logic's check against the reference, in 16 bits on the GPU
it is the eager 16-bit decoder the kernels are measured against.  The product never imports this file."""
import torch
import torch.nn.functional as F
from einops import rearrange

from tests import kernels_emul as E
from videosys_b200 import kernels


def unpack_conv_weight(w_packed, cin, cout, kt):
    """Inverse of kernels.pack_conv_weight: [cout, cin, kt, 3, 3]."""
    return w_packed[:cout, :, :cin].reshape(cout, kt, 3, 3, cin).permute(0, 4, 1, 2, 3)


def vae_conv3d(x, w_packed, bias, cout, kt, resid=None, round_conv=True):
    cin = x.shape[-1]
    w = unpack_conv_weight(w_packed, cin, cout, kt)
    xi = F.pad(x.permute(0, 4, 1, 2, 3), (1, 1, 1, 1))  # reference :131-132
    y = F.conv3d(xi, w) + bias.view(1, -1, 1, 1, 1) if round_conv else F.conv3d(xi, w, bias)
    if resid is not None:
        y = y + resid.permute(0, 4, 1, 2, 3)
    return y.permute(0, 2, 3, 4, 1).contiguous()


def vae_groupnorm_stats(x, groups, eps):
    B, C = x.shape[0], x.shape[-1]
    v = x.reshape(B, -1, groups, C // groups).transpose(1, 2).reshape(B, groups, -1).double()
    mean, var = v.mean(-1), v.var(-1, unbiased=False)
    return torch.stack([mean, (var + eps).rsqrt()], -1).float()


def _interp(z, size):
    """CogVideoXSpatialNorm3D's interpolation of zq (reference :166-174) on NCDHW."""
    T = size[0]
    if T > 1 and T % 2 == 1:
        first = F.interpolate(z[:, :, :1], size=(1, *size[1:]))
        rest = F.interpolate(z[:, :, 1:], size=(T - 1, *size[1:]))
        return torch.cat([first, rest], dim=2)
    return F.interpolate(z, size=size)


def vae_spatial_norm_silu(f, stats, gamma, beta, zyb, out, t_off=0):
    B, T, H, W, C = f.shape
    G = stats.shape[1]
    fi = f.permute(0, 4, 1, 2, 3)
    z = zyb.permute(0, 4, 1, 2, 3)
    zy, zb = _interp(z[:, :C], (T, H, W)), _interp(z[:, C:], (T, H, W))
    # F.group_norm on the GPU with the given statistics: mean and rstd kept in the input dtype, a = rstd * gamma,
    # b = -a * mean + beta, y = a * x + b in fp32
    mean = stats[..., 0].to(f.dtype).float().repeat_interleave(C // G, 1).view(B, C, 1, 1, 1)
    rstd = stats[..., 1].to(f.dtype).float().repeat_interleave(C // G, 1).view(B, C, 1, 1, 1)
    a = rstd * gamma.float().view(1, C, 1, 1, 1)
    n = (a * fi.float() + (beta.float().view(1, C, 1, 1, 1) - a * mean)).to(f.dtype)
    y = F.silu(n * zy + zb)
    out[:, t_off:t_off + T] = y.permute(0, 2, 3, 4, 1)
    return out


def vae_upsample2x(x, compress_time):
    """CogVideoXUpsample3D.forward before its conv (upsampling.py:40-60), channels-last."""
    xi = x.permute(0, 4, 1, 2, 3)
    if compress_time:
        if xi.shape[2] > 1 and xi.shape[2] % 2 == 1:
            first = F.interpolate(xi[:, :, 0], scale_factor=2.0)[:, :, None]
            rest = F.interpolate(xi[:, :, 1:], scale_factor=2.0)
            xi = torch.cat([first, rest], dim=2)
        elif xi.shape[2] > 1:
            xi = F.interpolate(xi, scale_factor=2.0)
        else:
            xi = F.interpolate(xi.squeeze(2), scale_factor=2.0)[:, :, None]
    else:
        b, c, t, h, w = xi.shape
        xi = F.interpolate(xi.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w), scale_factor=2.0)
        xi = xi.reshape(b, t, c, 2 * h, 2 * w).permute(0, 2, 1, 3, 4)
    return xi.permute(0, 2, 3, 4, 1).contiguous()


def vae_groupnorm_act(x, stats, gamma, beta, out=None, t_off=0, act=True):
    B, T, H, W, C = x.shape
    G = stats.shape[1]
    # F.group_norm on the GPU with the given statistics: mean and rstd kept in the input dtype, a = rstd * gamma,
    # b = -a * mean + beta, y = a * x + b in fp32
    mean = stats[..., 0].to(x.dtype).float().repeat_interleave(C // G, 1).view(B, 1, 1, 1, C)
    rstd = stats[..., 1].to(x.dtype).float().repeat_interleave(C // G, 1).view(B, 1, 1, 1, C)
    a = rstd * gamma.float()
    n = (a * x.float() + (beta.float() - a * mean)).to(x.dtype)
    # act = 1: x * torch.sigmoid(x) (Open-Sora-Plan's nonlinearity), act = 2: F.silu (nn.SiLU)
    y = F.silu(n) if act == 2 else n * torch.sigmoid(n) if act else n
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


def eager_attention(qkv, C, mixed):
    """The reference's bmm / scale / softmax / bmm on the (b*t, c, h*w) views (AttnBlock3D :920-932, Fix :387-411) of
    qkv [B, T, H, W, 3C] -> [B, T, H, W, C]."""
    B, T, H, W, _ = qkv.shape
    q, k, v = (_to_reference_frames(qkv[..., i * C:(i + 1) * C], mixed) for i in range(3))
    w_ = torch.bmm(q.permute(0, 2, 1), k) * (int(C) ** (-0.5))
    w_ = F.softmax(w_, dim=2)
    h_ = torch.bmm(v, w_.permute(0, 2, 1))  # (bt, c, hw)
    if mixed:
        return h_.reshape(B, C, T, H, W).permute(0, 2, 3, 4, 1)
    return h_.reshape(B, T, C, H, W).permute(0, 1, 3, 4, 2)


def vae_depth_to_time(x, out=None, t_off=0):
    y = rearrange(x.permute(0, 4, 1, 2, 3), "B (C ts) T H W -> B C (T ts) H W", ts=2).permute(0, 2, 3, 4, 1)
    if out is None:
        return y.contiguous()
    out[:, t_off:t_off + y.shape[1]] = y
    return out


NAMES = ["vae_conv3d", "vae_groupnorm_stats", "vae_spatial_norm_silu", "vae_upsample2x", "vae_groupnorm_act", "vae_upsample_linear2x",
         "vae_mix", "vae_attn_split", "vae_attn_softmax_", "vae_attn_merge", "vae_depth_to_time"]


def stand_ins():
    """name -> stand-in of every kernel entry the VAE decoders call (the eager 16-bit chain on the GPU)."""
    out = {n: globals()[n] for n in NAMES}
    out.update({n: getattr(E, n) for n in ("gemm_bias_act", "gemm_bias_residual")})
    return out


def emulate(monkeypatch):
    """tests/kernels_emul.emulate plus the VAE stand-ins, for the duration of one test."""
    E.emulate(monkeypatch)
    for n in NAMES:
        monkeypatch.setattr(kernels, n, globals()[n])
