"""TEST INFRASTRUCTURE ONLY -- torch/CPU stand-ins for the FP8 entries of ``videosys_b200.kernels`` (beside
tests/kernels_emul.py, whose stand-ins ``emulate`` also installs): quantization by the rule of tests/fp8_rule.py and the
GEMM as fake-quant -- the dequantized operands multiplied in fp32 -- rounded to the output dtype once."""
import torch
import torch.nn.functional as F

from tests import fp8_rule, kernels_emul
from videosys_b200 import kernels


def quant_rows_fp8(x):
    return fp8_rule.quant_rows(x)


def ln_modulate_fp8(x, mod, x_mask_u8, shift_row, scale_row, B, T, S, eps=1e-6):
    return fp8_rule.quant_rows(kernels_emul.ln_modulate(x, mod, x_mask_u8, shift_row, scale_row, B, T, S, eps=eps))


def _y(a, a_scale, w, w_scale, bias):
    a = a.view(torch.float8_e4m3fn) if a.dtype == torch.uint8 else a
    w = w.view(torch.float8_e4m3fn) if w.dtype == torch.uint8 else w
    y = fp8_rule.dequant(a, a_scale) @ fp8_rule.dequant(w, w_scale).T
    return y if bias is None else y + bias.float()


def gemm_fp8_bias_act(a, a_scale, w, w_scale, bias=None, act=0, out=None, dtype=torch.bfloat16):
    y = _y(a, a_scale, w, w_scale, bias).to(bias.dtype if bias is not None else dtype)
    if act == 1:
        y = F.gelu(y, approximate="tanh")
    if out is None:
        return y
    out.copy_(y.view(out.shape))
    return out


def gemm_fp8_bias_residual(a, a_scale, w, w_scale, bias, resid, mod=None, x_mask_u8=None, gate_row=-1, B=1, T=1, S=1, out=None):
    y = _y(a, a_scale, w, w_scale, bias).to(resid.dtype).reshape(resid.shape)
    out = resid if out is None else out
    if gate_row >= 0:
        return kernels_emul.gate_residual(resid, y, mod, x_mask_u8, gate_row, B, T, S, out=out)
    return kernels_emul.residual_add(resid, y, out=out)


NAMES = ["quant_rows_fp8", "ln_modulate_fp8", "gemm_fp8_bias_act", "gemm_fp8_bias_residual"]


def emulate(monkeypatch):
    kernels_emul.emulate(monkeypatch)
    g = globals()
    for n in NAMES:
        monkeypatch.setattr(kernels, n, g[n])
