"""TEST INFRASTRUCTURE ONLY -- torch/CPU stand-ins for the entries of ``videosys_b200.kernels``.

``-m "not gpu"`` tests patch these over the ctypes front end (``emulate(monkeypatch)``) to exercise the HOST logic of the
model mirrors -- buffer layouts, strides handed to the kernels, PAB bookkeeping, weight fusion, un-patchify -- against the
oracle in the authoring container, where no GPU exists.  Each stand-in takes exactly the arguments of the function it
replaces and honours the same pointer + stride conventions (``torch.as_strided`` on the storage behind the tensor the
caller passes).  The product never imports this file; on a GPU box the real kernels run (tests marked ``gpu``).
"""
import torch
import torch.nn.functional as F

from videosys_b200 import kernels


def _mod_row(mod, mask, row, B, T, C, dtype):
    """[B, T, 1, C] view of modulation row ``row`` with the per-frame t / t0 select."""
    m = mod.reshape(mod.shape[0], -1, mod.shape[-2], C)
    r0 = m[0, :B, row].view(B, 1, 1, C).expand(B, T, 1, C)
    if mask is None:
        return r0
    r1 = m[1, :B, row].view(B, 1, 1, C).expand(B, T, 1, C)
    return torch.where(mask.view(B, T, 1, 1).bool(), r0, r1)


def ln_modulate(x, mod, x_mask_u8, shift_row, scale_row, B, T, S, out=None, eps=1e-6, gamma=None, beta=None):
    C = x.shape[-1]
    xv = x.reshape(B, T, S, C)
    n = F.layer_norm(xv, (C,), gamma, beta, eps)
    y = n * (1 + _mod_row(mod, x_mask_u8, scale_row, B, T, C, x.dtype)) + _mod_row(mod, x_mask_u8, shift_row, B, T, C, x.dtype)
    y = y.reshape(x.shape)
    if out is None:
        return y.contiguous()
    out.copy_(y.view(out.shape))
    return out


def gate_residual(x, y, mod, x_mask_u8, gate_row, B, T, S, out=None, cache_out=None):
    C = x.shape[-1]
    g = _mod_row(mod, x_mask_u8, gate_row, B, T, C, x.dtype) * y.reshape(B, T, S, C)
    if cache_out is not None:
        cache_out.copy_(g.reshape(cache_out.shape))
    r = (x.reshape(B, T, S, C) + g).reshape(x.shape)
    if out is None:
        return r.contiguous()
    out.copy_(r)
    return out


def residual_add(x, y, out=None):
    r = x + y.reshape(x.shape)
    if out is None:
        return r
    out.copy_(r)
    return out


def gemm_bias_act(a, w, bias=None, act=0, out=None):
    y = F.linear(a, w, bias)
    if act == 1:
        y = F.gelu(y, approximate="tanh")
    if out is None:
        return y
    out.copy_(y.view(out.shape))
    return out


def gemm_bias_residual(a, w, bias, resid, mod=None, x_mask_u8=None, gate_row=-1, B=1, T=1, S=1, out=None):
    y = gemm_bias_act(a, w, bias).reshape(resid.shape)
    out = resid if out is None else out
    if gate_row >= 0:
        return gate_residual(resid, y, mod, x_mask_u8, gate_row, B, T, S, out=out)
    return residual_add(resid, y, out=out)


def _rope(x, cos, sin, pos):
    """x [..., D] at positions pos (long, broadcastable to x.shape[:-1]): interleaved pairs, fp32, cast back."""
    c, s = cos[pos], sin[pos]  # [..., D]
    xf = x.float()
    x1, x2 = xf[..., 0::2], xf[..., 1::2]
    rot = torch.stack((-x2, x1), -1).flatten(-2)
    return (xf * c + rot * s).to(x.dtype)


def qk_rmsnorm_(qkv, wq, wk, H, D, eps=1e-6, rope_cos=None, rope_sin=None, pos_div=1, pos_mod=1):
    rows = qkv.numel() // (3 * H * D)
    v = qkv.view(rows, 3, H, D)
    pos = (torch.arange(rows) // pos_div) % pos_mod
    for i, w in ((0, wq), (1, wk)):
        t = v[:, i]
        if w is not None:
            tf = t.float()
            t = w * (tf * torch.rsqrt(tf.pow(2).mean(-1, keepdim=True) + eps)).to(qkv.dtype)
        if rope_cos is not None:
            t = _rope(t, rope_cos, rope_sin, pos.view(rows, 1))
        v[:, i] = t
    return qkv


def qk_rope_halves_(qkv, rope_cos, rope_sin_signed, H, D, half, pos_div=1, pos_mod=1):
    rows = qkv.numel() // (3 * H * D)
    v = qkv.view(rows, 3, H, D)
    pos = (torch.arange(rows) // pos_div) % pos_mod
    c = rope_cos[pos].view(rows, 1, D).to(qkv.dtype)
    s = rope_sin_signed[pos].view(rows, 1, D).to(qkv.dtype)
    for i in (0, 1):
        t = v[:, i]
        blk = t.reshape(rows, H, D // (2 * half), 2, half)
        partner = blk.flip(3).reshape(rows, H, D)  # the other half of every rotation block
        v[:, i] = t * c + partner * s
    return qkv


def qk_layernorm_(qkv, wq, bq, wk, bk, H, D, eps=1e-6):
    rows = qkv.numel() // (3 * H * D)
    v = qkv.view(rows, 3, H, D)
    v[:, 0] = F.layer_norm(v[:, 0], (D,), wq, bq, eps)
    v[:, 1] = F.layer_norm(v[:, 1], (D,), wk, bk, eps)
    return qkv


def attn_short(qkv, wq, wk, rope_cos, rope_sin, n_outer, n_inner, outer_stride, inner_stride, tok_stride, n, H, D, scale,
               out=None, eps=1e-6, flags=0):
    rows = qkv.numel() // (3 * H * D)
    C = H * D
    flat = qkv.reshape(rows, 3, H, D)
    idx = (torch.arange(n_outer).view(-1, 1, 1) * outer_stride + torch.arange(n_inner).view(1, -1, 1) * inner_stride
           + torch.arange(n).view(1, 1, -1) * tok_stride).reshape(-1, n)  # [seqs, n] row indices
    g = flat[idx]  # [seqs, n, 3, H, D]
    q, k, v = g[:, :, 0], g[:, :, 1], g[:, :, 2]
    if not flags & 1:
        def rms(t, w):
            tf = t.float()
            return w * (tf * torch.rsqrt(tf.pow(2).mean(-1, keepdim=True) + eps)).to(t.dtype)
        q, k = rms(q, wq), rms(k, wk)
    if rope_cos is not None:
        pos = torch.arange(n).view(1, n, 1)
        q, k = _rope(q, rope_cos, rope_sin, pos), _rope(k, rope_cos, rope_sin, pos)
    q, k, v = (t.transpose(1, 2) for t in (q, k, v))  # [seqs, H, n, D]
    if n == 1:
        o = v
    elif flags & 2:
        o = F.scaled_dot_product_attention(q, k, v, scale=scale)
    else:  # native_attention (attentions.py:111-120)
        a = ((q * scale) @ k.transpose(-2, -1)).to(torch.float32).softmax(-1).to(q.dtype)
        o = a @ v
    o = o.transpose(1, 2).reshape(-1, n, C)
    out = torch.empty(rows, C, dtype=qkv.dtype) if out is None else out
    out.view(rows, C)[idx.reshape(-1)] = o.reshape(-1, C)
    return out


def _strided(t, sizes, strides):
    return torch.as_strided(t, sizes, strides, t.storage_offset())


def attn_flash(q, k, v, nb, nq, nk, H, D, q_row_stride, q_batch_stride, kv_row_stride, kv_batch_stride, scale, kv_lens=None,
               out=None, out_row_stride=None, out_batch_stride=None):
    qv = _strided(q, (nb, H, nq, D), (q_batch_stride, D, q_row_stride, 1))
    kv = _strided(k, (nb, H, nk, D), (kv_batch_stride, D, kv_row_stride, 1))
    vv = _strided(v, (nb, H, nk, D), (kv_batch_stride, D, kv_row_stride, 1))
    mask = None
    if kv_lens is not None:
        mask = (torch.arange(nk).view(1, 1, 1, nk) < torch.tensor(list(kv_lens)).view(nb, 1, 1, 1))
    o = F.scaled_dot_product_attention(qv, kv, vv, attn_mask=mask, scale=scale)  # [nb, H, nq, D]
    if out is None:
        out = torch.empty(nb, nq, H * D, dtype=q.dtype)
    ors = H * D if out_row_stride is None else out_row_stride
    obs = nq * H * D if out_batch_stride is None else out_batch_stride
    _strided(out, (nb, H, nq, D), (obs, D, ors, 1)).copy_(o)
    return out


def modulation_table(table, t, t0):
    rows, C = table.shape
    B = t.shape[0]
    m0 = table[None] + t.reshape(B, rows, C)
    m1 = m0 if t0 is None else table[None] + t0.reshape(B, rows, C)
    return torch.stack([m0, m1], 0).contiguous()


def patch_embed(*a, **k):
    return None  # "shape not taken": the callers run their torch convolution


def require_cuda(t, what="vsb200", half_only=False):
    return None


NAMES = ["ln_modulate", "gate_residual", "residual_add", "gemm_bias_act", "gemm_bias_residual", "qk_rmsnorm_", "qk_rope_halves_", "qk_layernorm_",
         "attn_short", "attn_flash", "modulation_table", "patch_embed", "require_cuda"]


def emulate(monkeypatch):
    """Patch the stand-ins over ``videosys_b200.kernels`` for the duration of one test."""
    g = globals()
    for n in NAMES:
        monkeypatch.setattr(kernels, n, g[n])


def emulate_global():
    """The same for a spawned worker process (no monkeypatch fixture there; the process ends with the test)."""
    g = globals()
    for n in NAMES:
        setattr(kernels, n, g[n])
