"""TEST INFRASTRUCTURE ONLY -- a torch stand-in for the OpenSora v1.2 VAE encoder's strided entry ``vae_conv_down``, on
top of tests/kernels_emul_vae.py.  It takes exactly the arguments of the function it replaces, with its channels-last
layout and packed weight, and computes what the reference's eager chain computes: Downsample2D's F.pad(x, (0, 1, 0, 1))
and a stride-2 F.conv2d per frame (kt = 1), or CausalConv3d's F.pad (one zero frame in front, spatial padding 1) and
F.conv3d with stride (2, 1, 1) (kt = 3).  The product never imports this file."""
import torch.nn.functional as F

from tests import kernels_emul_vae
from videosys_b200 import kernels


def vae_conv_down(x, w_packed, bias, cout, kt, round_conv=True):
    w = kernels_emul_vae.unpack_conv_weight(w_packed, x.shape[-1], cout, kt)
    xi = x.permute(0, 4, 1, 2, 3)
    if kt == 1:
        xi, stride = F.pad(xi, (0, 1, 0, 1)), (1, 2, 2)
    else:
        xi, stride = F.pad(xi, (1, 1, 1, 1, 1, 0)), (2, 1, 1)
    y = F.conv3d(xi, w, stride=stride) + bias.view(1, -1, 1, 1, 1) if round_conv else F.conv3d(xi, w, bias, stride=stride)
    return y.permute(0, 2, 3, 4, 1).contiguous()


NAMES = ["vae_conv_down"]


def stand_ins():
    """kernels_emul_vae.stand_ins() plus the encoder's strided entry."""
    out = kernels_emul_vae.stand_ins()
    out.update({n: globals()[n] for n in NAMES})
    return out


def emulate(monkeypatch):
    kernels_emul_vae.emulate(monkeypatch)
    for n in NAMES:
        monkeypatch.setattr(kernels, n, globals()[n])
