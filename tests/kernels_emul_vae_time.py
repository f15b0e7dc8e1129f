"""TEST INFRASTRUCTURE ONLY -- torch stand-ins for the SVD temporal decoder's kernel entries (``vae_conv_time``,
``vae_time_conv_rgb``), on top of tests/kernels_emul_vae.py.  Each takes the arguments of the function it replaces and
computes what the reference's eager chain computes (F.conv3d on NCDHW with the (3, 1, 1) kernel, + bias, + input, the
AlphaBlender's products and sum as 16-bit tensor ops), on whatever device and dtype the tensors have.  The product never
imports this file."""
import torch
import torch.nn.functional as F

from tests import kernels_emul_vae
from videosys_b200 import kernels


def vae_conv_time(x, w_packed, bias, cout, kt, resid=None, mix=None, round_conv=True):
    cin = x.shape[-1]
    w = w_packed[:cout, :, :cin].permute(0, 2, 1)[..., None, None]  # [cout, cin, kt, 1, 1]
    xi = x.permute(0, 4, 1, 2, 3)
    y = (F.conv3d(xi, w) + bias.view(1, -1, 1, 1, 1) if round_conv else F.conv3d(xi, w, bias)).permute(0, 2, 3, 4, 1)
    if mix is not None:  # TemporalResnetBlock: input_tensor + hidden_states; AlphaBlender: alpha * x + (1 - alpha) * t
        a, b = (torch.tensor([m], dtype=y.dtype, device=y.device) for m in mix)
        return (a * resid + b * (resid + y)).contiguous()
    if resid is not None:
        y = y + resid
    return y.contiguous()


def vae_time_conv_rgb(x, weight, bias):
    y = F.conv3d(x.permute(0, 4, 1, 2, 3), weight, padding=(1, 0, 0)) + bias.view(1, -1, 1, 1, 1)
    return y.permute(0, 2, 3, 4, 1).contiguous()


NAMES = ["vae_conv_time", "vae_time_conv_rgb"]


def stand_ins():
    """kernels_emul_vae.stand_ins() plus the temporal decoder's entries."""
    out = kernels_emul_vae.stand_ins()
    out.update({n: globals()[n] for n in NAMES})
    return out


def emulate(monkeypatch):
    kernels_emul_vae.emulate(monkeypatch)
    for n in NAMES:
        monkeypatch.setattr(kernels, n, globals()[n])
