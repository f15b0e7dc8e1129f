"""The attention layouts the model front ends share, on the vsb200 kernels.

Every function works on the packed projection buffers the front ends already hold (no copies into another layout) and
hands the kernels strided views of them.  The kernels are looked up on ``kernels`` at call time.

RoPE tables come in two formats, told apart by their length:
  * ``(cos, sin)`` fp32 [positions, head_dim]: rotation of interleaved pairs (2i, 2i+1), the pairing of
    ``vsb_qk_rmsnorm_rope`` and ``vsb_attn_short``;
  * ``(cos, sin_signed, half)``: half-rotation blocks of ``half`` channels (``vsb_qk_rope_halves``), the sign of
    rotate_half folded into the sin table.
"""
import torch

from ... import kernels
from ...core.distributed import comm


def _flags(wq, sdpa):
    """attn_short flags: bit 0 = no q / k RMSNorm, bit 1 = SDPA rounding (else native_attention's)."""
    return (1 if wq is None else 0) | (2 if sdpa else 0)


def apply_rope_(qkv, rope, H, D, pos_div=1, pos_mod=1):
    """RoPE in place on q and k of a packed [rows, 3, H, D] buffer; row r takes table row (r // pos_div) % pos_mod."""
    if len(rope) == 2:
        kernels.qk_rmsnorm_(qkv, None, None, H, D, rope_cos=rope[0], rope_sin=rope[1], pos_div=pos_div, pos_mod=pos_mod)
    else:
        kernels.qk_rope_halves_(qkv, rope[0], rope[1], H, D, rope[2], pos_div=pos_div, pos_mod=pos_mod)
    return qkv


def temporal_attention(qkv, B, T, S, H, D, scale, short_max, wq=None, wk=None, rope=None, sdpa=False):
    """Self-attention over the T frames at every (sample, patch) of the token-major qkv [B, T, S, 3, H, D]; returns
    [B*T*S, H*D] in the same order.  wq / wk: per-head RMSNorm of q / k; rope: table indexed by the frame.

    T <= short_max: one ``attn_short`` launch (norm and interleaved RoPE inside the kernel).  Longer: the norm / RoPE
    pre-pass, then one ``attn_flash`` per sample over strided views (batch = patch, row = frame)."""
    if rope is not None and len(rope) == 3:  # attn_short only rotates interleaved pairs
        apply_rope_(qkv, rope, H, D, pos_div=S, pos_mod=T)
        rope = None
    cos, sin = rope if rope is not None else (None, None)
    if T <= short_max:
        return kernels.attn_short(qkv.view(-1, 3, H, D), wq, wk, cos, sin, B, S, T * S, 1, S, T, H, D, scale,
                                  flags=_flags(wq, sdpa))
    if S > 65535:
        raise RuntimeError("temporal flash attention: more than 65535 patches per frame")
    if wq is not None or cos is not None:
        kernels.qk_rmsnorm_(qkv, wq, wk, H, D, rope_cos=cos, rope_sin=sin, pos_div=S, pos_mod=T)
    C = H * D
    o = torch.empty(B * T * S, C, dtype=qkv.dtype, device=qkv.device)
    q3 = qkv.view(B, T * S, 3, C)
    for b in range(B):
        kernels.attn_flash(q3[b, :, 0], q3[b, :, 1], q3[b, :, 2], S, T, T, H, D, S * 3 * C, 3 * C, S * 3 * C, 3 * C, scale,
                           out=o[b * T * S:], out_row_stride=S * C, out_batch_stride=C)
    return o


def temporal_cross_attention(q, kv, B, T, Tk, S, H, D, scale):
    """Attention over frames at every (sample, patch) with fewer key frames than query frames: q [B*T*S, H*D] token-major,
    kv [B*Tk*S, 2, H*D] (packed k | v, token-major over Tk frames).  One ``attn_flash`` per sample over strided views
    (batch = patch, q row = frame, kv row = key frame).  Returns [B*T*S, H*D] in the order of q."""
    if S > 65535:
        raise RuntimeError("temporal flash attention: more than 65535 patches per frame")
    C = H * D
    q = q.view(B * T * S, C)
    o = torch.empty(B * T * S, C, dtype=q.dtype, device=q.device)
    for b in range(B):
        kvb = kv[b * Tk * S:]
        kernels.attn_flash(q[b * T * S:], kvb[:, 0], kvb[:, 1], S, T, Tk, H, D, S * C, C, S * 2 * C, 2 * C, scale,
                           out=o[b * T * S:], out_row_stride=S * C, out_batch_stride=C)
    return o


def packed_self_attention(qkv, nb, n, H, D, scale, short_max=None, wq=None, wk=None, sdpa=False):
    """Self-attention of nb sequences of n tokens in one packed [nb*n, 3, H, D] buffer; returns [nb, n, H*D].
    n <= short_max runs ``attn_short`` (q / k norm inside the kernel); otherwise the norm pass (when wq is given) and
    ``attn_flash``.  short_max=None always takes the flash kernel."""
    if short_max is not None and n <= short_max:
        return kernels.attn_short(qkv.view(-1, 3, H, D), wq, wk, None, None, nb, 1, n, 0, 1, n, H, D, scale,
                                  flags=_flags(wq, sdpa))
    if wq is not None:
        kernels.qk_rmsnorm_(qkv, wq, wk, H, D)
    C = H * D
    q3 = qkv.view(-1, 3, C)
    return kernels.attn_flash(q3[:, 0], q3[:, 1], q3[:, 2], nb, n, n, H, D, 3 * C, n * 3 * C, 3 * C, n * 3 * C, scale)


def cross_attention(q, kv, nb, nq, nk, H, D, scale, kv_lens=None):
    """q [nb*nq, H*D] against the keys / values in the last two slots of kv [nb*nk, m, H*D] (m = 2: packed k | v, m = 3:
    q | k | v); kv_lens: valid keys per sample (a prefix).  Returns [nb, nq, H*D]."""
    C = H * D
    m = kv.shape[1]
    return kernels.attn_flash(q, kv[:, -2], kv[:, -1], nb, nq, nk, H, D, C, nq * C, m * C, nk * m * C, scale, kv_lens=kv_lens)


def ulysses_attention(qkv5, n_text, n_valid, sp_group, scale, rope=None):
    """Head-scatter sequence-parallel self-attention.  qkv5 [B, n_text + Nl, 3, H, D]: the replicated text rows and
    this rank's chunk of the other rows.  The exchange (``comm.ulysses_scatter_heads``) gives every row for H / sp heads;
    rows from n_valid on are padding: they are not keys and their output is zero.  rope: table over the gathered rows.
    Returns [B, n_text + Nl, H*D]: this rank's rows, every head."""
    full = comm.ulysses_scatter_heads(qkv5, n_text, sp_group)
    B, Lf, _, Hn, D = full.shape
    Cn = Hn * D
    if rope is not None:
        apply_rope_(full, rope, Hn, D, pos_div=1, pos_mod=Lf)
    f3 = full.view(B * Lf, 3, Cn)
    of = torch.empty(B, Lf, Cn, dtype=full.dtype, device=full.device)
    if Lf > n_valid:
        of[:, n_valid:].zero_()
    kernels.attn_flash(f3[:, 0], f3[:, 1], f3[:, 2], B, n_valid, n_valid, Hn, D, 3 * Cn, Lf * 3 * Cn, 3 * Cn, Lf * 3 * Cn, scale,
                       out=of, out_row_stride=Cn, out_batch_stride=Lf * Cn)
    return comm.ulysses_gather_heads(of, n_text, sp_group).contiguous()
