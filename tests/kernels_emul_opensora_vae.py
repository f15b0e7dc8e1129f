"""TEST INFRASTRUCTURE ONLY -- torch stand-ins for the OpenSora v1.2 VAE decoder entries of ``videosys_b200.kernels``, on
top of the stand-ins of tests/kernels_emul_osp_vae.py (and through it tests/kernels_emul_vae.py): ``vae_groupnorm_act`` with
act = 2 (F.group_norm, then F.silu as nn.SiLU computes it) and ``vae_depth_to_time`` (the reference's einops rearrange).
Each takes exactly the arguments of the function it replaces, with the kernels' channels-last layouts, on whatever device
and dtype the tensors have.  The product never imports this file."""
import torch.nn.functional as F
from einops import rearrange

from tests import kernels_emul as E
from tests import kernels_emul_osp_vae as EO
from tests import kernels_emul_vae as EV
from videosys_b200 import kernels


def vae_groupnorm_act(x, stats, gamma, beta, out=None, t_off=0, act=True):
    if act != 2:
        return EO.vae_groupnorm_act(x, stats, gamma, beta, out=out, t_off=t_off, act=act)
    y = F.silu(EO.vae_groupnorm_act(x, stats, gamma, beta, act=False))
    if out is None:
        return y.contiguous()
    out[:, t_off:t_off + y.shape[1]] = y
    return out


def vae_depth_to_time(x, out=None, t_off=0):
    y = rearrange(x.permute(0, 4, 1, 2, 3), "B (C ts) T H W -> B C (T ts) H W", ts=2).permute(0, 2, 3, 4, 1)
    if out is None:
        return y.contiguous()
    out[:, t_off:t_off + y.shape[1]] = y
    return out


NAMES = ["vae_groupnorm_act", "vae_depth_to_time"]


def stand_ins():
    """name -> stand-in of every kernel entry the OpenSora VAE decoder calls (the eager 16-bit chain on the GPU)."""
    out = {n: getattr(mod, n) for mod, names in ((EV, EV.NAMES), (EO, EO.NAMES)) for n in names}
    out.update({n: getattr(E, n) for n in ("gemm_bias_act", "gemm_bias_residual")})
    out.update({n: globals()[n] for n in NAMES})
    return out


def emulate(monkeypatch):
    """tests/kernels_emul_osp_vae.emulate plus the OpenSora v1.2 VAE stand-ins, for the duration of one test."""
    EO.emulate(monkeypatch)
    for n in NAMES:
        monkeypatch.setattr(kernels, n, globals()[n])
