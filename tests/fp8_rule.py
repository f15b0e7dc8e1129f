"""TEST INFRASTRUCTURE ONLY -- the e4m3 quantization rule of include/vsb200.h restated in torch (CPU or GPU tensors).

A row x of 16-bit values has amax = max |x|.  amax > 0: codes = float8_e4m3fn(fp32(x) * s) with s = fp32(448 / amax)
(torch rounds to nearest even, as cvt.rn.satfinite.e4m3x2.f32 does inside the finite range), scale = fp32(amax / 448).
amax == 0: all-zero codes and scale 1."""
import torch


def quant_rows(x):
    """(codes float8_e4m3fn [..., K], scale fp32 [...]) of x [..., K]."""
    xf = x.float()
    amax = xf.abs().amax(-1, keepdim=True)
    nz = amax > 0
    s = torch.where(nz, torch.full_like(amax, 448.0) / torch.where(nz, amax, torch.ones_like(amax)), torch.zeros_like(amax))
    q = (xf * s).to(torch.float8_e4m3fn)
    q = torch.where(nz, q.view(torch.uint8), torch.zeros_like(q.view(torch.uint8))).view(torch.float8_e4m3fn)
    scale = torch.where(nz, amax / 448.0, torch.ones_like(amax)).squeeze(-1)
    return q, scale


def dequant(q, scale):
    """float32 q * scale per row (exact: a 4-bit significand times an fp32 scale)."""
    return q.float() * scale.float().unsqueeze(-1)


def fake_quant_linear(x, w, bias):
    """The FP8 Linear on fp32 arithmetic: both operands quantized per row by the rule, products of the dequantized values
    summed in fp32, + bias."""
    qa, sa = quant_rows(x)
    qw, sw = quant_rows(w)
    y = dequant(qa, sa) @ dequant(qw, sw).T
    return y if bias is None else y + bias.float()
