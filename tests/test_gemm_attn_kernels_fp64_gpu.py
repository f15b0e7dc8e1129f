"""The GEMM (csrc/gemm_wgmma.cu) and attention kernels (csrc/attn_wgmma.cu, csrc/attn_mma.cu, csrc/attn_short.cu) element
by element against float64, in bf16 and fp16, under the acceptance rule of tests/vae_fp64.py with the reference chains of
tests/gemm_attn_fp64.py.

Every check prints eps, the bit-equal fraction, the largest error in ulps, the accepted flips with their largest distance
to the midpoint, the count outside the legal set, and the fraction of elements with more than one legal value.  Inputs
look like hidden states (a DC offset and four channels x 20).  Every arithmetic kernel is launched twice and the two
results compared bit for bit (NaN included).  The float64 references run on the GPU.

Which case reaches which template instance and dispatch branch:
  gemm_tile_kernel<192, 0>     act 0, N % 192 == 0 or (N > 192 and N % 128 != 0)   N = 200, 520, 6912, 1152, 3456, 1920
  gemm_tile_kernel<128, 0>     act 0, otherwise                                     N = 8, 64, 136
  gemm_wgmma_kernel<1>, <3>    GELU at K <= 1536                                    K = 8 .. 1536, the exhaustive GELU cases
  gemm_tile_kernel<., 1>, <., 3>  GELU at K > 1536                                  K = 1544, 4608, 1920 (CogVideoX), 2304 (OSP)
  gemm_wgmma_kernel<2>         every residual epilogue                              gate rows 2 / 5 and the plain add
  attn_wgmma_kernel<64>, <72>  head_dim 64 / 72 (128-key tiles)
  attn_mma_kernel<32>, <48>, <80>, <96>, <128>   the other head dims (64-key tiles)
  attn_short_kernel<64 | 72, 32>   n <= 32;   attn_short_kernel<64 | 72, 64>   33 <= n <= 64"""
import pytest
import torch
import torch.nn.functional as F

from tests import gemm_attn_fp64 as G
from tests import vae_fp64 as V
from tests.test_dit_kernels_fp64_gpu import _masks
from videosys_b200 import kernels
from videosys_b200._lib import VsbError

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]
IDS = ["bf16", "fp16"]
both = pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
EPI = {0: 0, 1: 1, 3: 2}  # kernel epilogue -> public act of gemm_bias_act


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _rand(*shape, dtype, scale=1.0, offset=0.0, seed=0):
    return (offset + scale * torch.randn(*shape, generator=_gen(seed))).to(dtype).to(DEV)


def _hidden(*shape, dtype, seed, offset=0.3, scale=1.0):
    """Hidden-state-like values, channels last: a DC offset and four massive channels (x 20)."""
    z = offset + torch.randn(*shape, generator=_gen(seed))
    z[..., 3:7] *= 20
    return (scale * z).to(dtype).to(DEV)


def _check(what, got, chain, mask=None):
    ok, _ = V.check(what, got, chain, mask)
    G.legal_report(chain if mask is None else chain.take(mask))
    return ok


def _twice(what, fn):
    a = fn()
    b = fn()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{what}: two launches differ"  # NaN bits included
    return a


# =====================================================================================================================
# GEMM
# =====================================================================================================================
def _gemm_inputs(M, N, K, dtype, seed=0):
    a = _hidden(M, K, dtype=dtype, seed=seed + 1)
    w = _rand(N, K, dtype=dtype, scale=K**-0.5, seed=seed + 2)
    bias = _rand(N, dtype=dtype, scale=0.5, seed=seed + 3)
    return a, w, bias


def _gemm_run(what, a, w, bias, act, rows=None):
    got = _twice(what, lambda: kernels.gemm_bias_act(a, w, bias, EPI[act]))
    if rows is None:
        return _check(what, got, G.gemm_chain(a, w, bias, act))
    return _check(what, got[rows], G.gemm_chain(a[rows], w, bias, act))


@both
@pytest.mark.parametrize("act", [0, 1, 3], ids=["none", "tanh", "erf"])
def test_gemm_shapes_fp64(act, dtype):
    """M in {1, 127, 128, 129, 300} x N in {8, 64, 136, 200, 520, 6912} x K in {8, 24, 64, 72, 1152, 4608} (the largest
    products on fewer rows), with and without bias; K < 64 is a single partial k-block."""
    failed = []
    for K in (8, 24, 64, 72, 1152, 4608):
        for N in (8, 64, 136, 200, 520, 6912):
            for M in (1, 127, 128, 129, 300):
                if N * K > 1 << 22 and M not in (1, 129):
                    continue
                a, w, bias = _gemm_inputs(M, N, K, dtype, seed=K + N)
                bb = None if (M + N) % 3 == 0 else bias
                what = f"gemm act={act} {dtype} M={M} N={N} K={K} bias={bb is not None}"
                if not _gemm_run(what, a, w, bb, act):
                    failed.append(what)
    assert not failed, failed


@both
@pytest.mark.parametrize("act", [1, 3], ids=["tanh", "erf"])
@pytest.mark.parametrize("K", [1536, 1544])
def test_gemm_gelu_kernel_boundary_fp64(K, act, dtype):
    """K = 1536 is the longest GELU GEMM on the persistent kernel, K = 1544 the shortest on the tile kernel."""
    failed = []
    for M, N in ((129, 1152), (300, 520)):
        a, w, bias = _gemm_inputs(M, N, K, dtype, seed=K)
        what = f"gemm act={act} {dtype} M={M} N={N} K={K}"
        if not _gemm_run(what, a, w, bias, act):
            failed.append(what)
    assert not failed, failed


MODEL_GEMMS = {
    # name: (dtypes, M, N, K, act)
    "OpenSora qkv 1152->3456": (DTYPES, 2048, 3456, 1152, 0),
    "OpenSora fc1 1152->4608 tanh": (DTYPES, 2048, 4608, 1152, 1),
    "OpenSora fc2 4608->1152": (DTYPES, 2048, 1152, 4608, 0),
    "CogVideoX-2b fc1 1920->7680 tanh": ([torch.float16], 1350, 7680, 1920, 1),
    "CogVideoX-2b fc2 7680->1920": ([torch.float16], 1350, 1920, 7680, 0),
    "Open-Sora-Plan v1.2.0 2304->9216 erf": (DTYPES, 1200, 9216, 2304, 3),
}


@pytest.mark.parametrize("name", list(MODEL_GEMMS))
def test_gemm_model_shapes_fp64(name):
    """Model widths at a few thousand rows; the reference on the first, a middle and the last row tile."""
    dtypes, M, N, K, act = MODEL_GEMMS[name]
    rows = torch.cat([torch.arange(0, 128), torch.arange(M // 2, M // 2 + 64), torch.arange(M - 128, M)]).to(DEV)
    failed = []
    for dtype in dtypes:
        a, w, bias = _gemm_inputs(M, N, K, dtype, seed=N)
        what = f"gemm {name} {dtype} M={M}"
        if not _gemm_run(what, a, w, bias, act, rows):
            failed.append(what)
    assert not failed, failed


@both
@pytest.mark.parametrize("act", [0, 1, 3], ids=["none", "tanh", "erf"])
def test_gemm_cancellation_fp64(act, dtype):
    """A DC-offset A against zero-mean W rows at K = 4608: the partial sums run far above the result, which is what the
    truncation eps is there for."""
    M, N, K = 129, 520, 4608
    a = _hidden(M, K, dtype=dtype, seed=31, offset=8.0)
    w = torch.randn(N, K, generator=_gen(32)) * K**-0.5
    w = w - w.mean(1, keepdim=True)
    w[:, 3:7] = 0
    w = w.to(dtype).to(DEV)
    bias = _rand(N, dtype=dtype, scale=0.5, seed=33)
    assert _gemm_run(f"gemm cancellation act={act} {dtype}", a, w, bias, act)


def _all_finite_values(dtype):
    allv = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype)
    x = allv[torch.isfinite(allv.float())]
    return torch.cat([x, torch.zeros((-x.numel()) % 8, dtype=dtype)]).to(DEV)


@both
@pytest.mark.parametrize("act", [1, 3], ids=["tanh", "erf"])
@pytest.mark.parametrize("K", [8, 1544], ids=["persistent", "tile"])
def test_gemm_gelu_every_16_bit_value(K, act, dtype):
    """One-hot A (row 0 = e0), bias 0: out[0, n] = act(w[n, 0]) for every finite 16-bit value.  fp16 adds a row e0 + e1
    with w[:, 1] = w[:, 0], whose two-term sums overflow to +-inf for the largest values: non-finite pre-activations must
    give what torch's fp32 F.gelu gives."""
    x = _all_finite_values(dtype)
    N = x.numel()
    rows = 2 if dtype == torch.float16 else 1
    a = torch.zeros(rows, K, dtype=dtype, device=DEV)
    a[:, 0] = 1
    w = torch.zeros(N, K, dtype=dtype, device=DEV)
    w[:, 0] = x
    if rows == 2:
        a[1, 1] = 1
        w[:, 1] = x
    what = f"gelu act={act} {dtype} K={K} every value"
    got = _twice(what, lambda: kernels.gemm_bias_act(a, w, None, EPI[act]))
    pre = V.round16(a.double() @ w.double().T, dtype)  # exact: at most two terms
    fin = torch.isfinite(pre)
    ok = _check(what, got, G.gemm_chain(a, w, None, act), fin)
    want = F.gelu(pre.float(), approximate="tanh" if act == 1 else "none")
    g = got.float()
    nonfin = ~fin
    if bool(nonfin.any()):
        same = (torch.isnan(g) & torch.isnan(want)) | (g == want)
        print(f"    {int(nonfin.sum())} non-finite pre-activations: {int((~same[nonfin]).sum())} differ from torch's fp32 F.gelu")
        ok = ok and bool(same[nonfin].all())
    assert ok


def _guarded(rows, C, dtype):
    buf = torch.full((rows + 2, C), float("nan"), dtype=dtype, device=DEV)
    return buf, buf[1:-1]


def _guards_intact(what, buf):
    assert bool(torch.isnan(buf[0].float()).all() and torch.isnan(buf[-1].float()).all()), f"{what}: wrote outside its output"


@both
@pytest.mark.parametrize("gate_row", [2, 5, -1], ids=["gate2", "gate5", "plain"])
def test_gemm_residual_epilogue_fp64(gate_row, dtype):
    """Every mask pattern, each gate row the models use and the plain add; in place, and out != resid (resid unchanged);
    output rows past M are NaN guard rows that must stay untouched."""
    failed = []
    for (B, T, S), N, K in (((2, 3, 50), 1152, 1152), ((1, 2, 1), 520, 72), ((2, 4, 33), 136, 4608)):
        M = B * T * S
        a, w, bias = _gemm_inputs(M, N, K, dtype, seed=N + K)
        resid = _hidden(M, N, dtype=dtype, seed=5)
        mod = _rand(2, B, 6, N, dtype=dtype, scale=0.5, seed=6)
        for mname, mask in _masks(B, T).items():
            if gate_row < 0 and mname != "none":
                continue
            what = f"gemm residual {dtype} gate_row={gate_row} M={M} N={N} K={K} mask={mname}"
            ch = G.gemm_residual_chain(a, w, bias, resid, mod, mask, gate_row, B, T, S)
            r0 = resid.clone()
            buf, out = _guarded(M, N, dtype)
            kernels.gemm_bias_residual(a, w, bias, resid, mod, mask, gate_row, B, T, S, out=out)
            _guards_intact(what, buf)
            assert torch.equal(resid, r0), f"{what}: resid changed"
            again = kernels.gemm_bias_residual(a, w, bias, resid, mod, mask, gate_row, B, T, S, out=torch.empty_like(resid))
            assert torch.equal(out, again), f"{what}: two launches differ"
            if not _check(what, out.view(B, T, S, N), ch):
                failed.append(what)
            ibuf, inner = _guarded(M, N, dtype)
            inner.copy_(resid)
            kernels.gemm_bias_residual(a, w, bias, inner, mod, mask, gate_row, B, T, S)  # in place, as the models call it
            _guards_intact(what + " in place", ibuf)
            assert torch.equal(inner, out), f"{what}: in place differs"
    assert not failed, failed


# =====================================================================================================================
# flash attention
# =====================================================================================================================
QK_SCALE = 0.25  # q and k as hidden states times 1/4 (exact): scores of a few units, as after the models' q / k norms


def _qkv(nb, n, H, D, dtype, seed, offset=0.3):
    x = _hidden(nb, n, 3, H, D, dtype=dtype, seed=seed, offset=offset)
    x[:, :, :2] *= QK_SCALE
    return x


def _q(nb, nq, H, D, dtype, seed):
    return _hidden(nb, nq, H, D, dtype=dtype, seed=seed, scale=QK_SCALE)


def _kv(nb, nk, H, D, dtype, seed):
    kv = _hidden(nb, nk, 2, H, D, dtype=dtype, seed=seed)
    kv[:, :, 0] *= QK_SCALE
    return kv


def _flash_packed(qkv, lens=None):
    nb, n, _, H, D = qkv.shape
    C = H * D
    return lambda: kernels.attn_flash(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], nb, n, n, H, D, 3 * C, n * 3 * C, 3 * C,
                                      n * 3 * C, D**-0.5, kv_lens=lens)


def _flash_cross(q, kv, lens=None):
    nb, nq, H, D = q.shape
    nk = kv.shape[1]
    C = H * D
    return lambda: kernels.attn_flash(q, kv[:, :, 0], kv[:, :, 1], nb, nq, nk, H, D, C, nq * C, 2 * C, nk * 2 * C, D**-0.5,
                                      kv_lens=lens)


def _flash_check(what, fn, q, k, v, lens=None, rows=None, heads=None):
    got = _twice(what, fn).view(q.shape[0], q.shape[1], q.shape[2], q.shape[3])
    hs = slice(None) if heads is None else slice(0, heads)
    ch = G.flash_chain(q[:, :, hs], k[:, :, hs], v[:, :, hs], q.shape[-1] ** -0.5, lens, rows=rows)
    g = got[:, :, hs] if rows is None else got[:, rows][:, :, hs]
    return _check(what, g, ch)


HEAD_DIMS = [64, 72, 32, 48, 80, 96, 128]


@both
@pytest.mark.parametrize("D", HEAD_DIMS)
def test_attn_flash_lengths_fp64(D, dtype):
    """Self-attention (packed qkv) at every tile edge: nk = nq in {1, 63, 64, 65, 127, 128, 129}, and cross-attention
    nq in {1, 16, 127, 128, 129, 272} against nk in {1, 63, 65, 129, 3600}."""
    H = 2
    failed = []
    for n in (1, 63, 64, 65, 127, 128, 129):
        qkv = _qkv(2, n, H, D, dtype, seed=n)
        what = f"attn_flash self D={D} {dtype} n={n}"
        if not _flash_check(what, _flash_packed(qkv), qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]):
            failed.append(what)
    for nq, nk in ((1, 129), (16, 1), (127, 63), (128, 65), (129, 3600), (272, 129)):
        q = _q(2, nq, H, D, dtype, seed=nq)
        kv = _kv(2, nk, H, D, dtype, seed=nk + 1)
        what = f"attn_flash cross D={D} {dtype} nq={nq} nk={nk}"
        if not _flash_check(what, _flash_cross(q, kv), q, kv[:, :, 0], kv[:, :, 1]):
            failed.append(what)
    assert not failed, failed


@both
@pytest.mark.parametrize("D", [72, 96], ids=["wgmma", "mma"])
def test_attn_flash_layouts_fp64(D, dtype):
    """kv_lens with 1, nk and 64 batches (the kAttnMaxLens limit); more work items than SMs; strided output (the temporal
    path over >= 30 frames, rows S * C apart, written into a NaN-guarded token-major buffer)."""
    failed = []
    H = 2
    for nb, nq, nk in ((1, 40, 300), (3, 129, 300), (64, 16, 200)):
        lens = [1 + (37 * b + nk - 1) % nk for b in range(nb)]
        lens[0] = nk
        if nb > 1:
            lens[1] = 1
        q = _q(nb, nq, H, D, dtype, seed=nb)
        kv = _kv(nb, nk, H, D, dtype, seed=nb + 1)
        what = f"attn_flash lens D={D} {dtype} nb={nb} nq={nq} nk={nk}"
        if not _flash_check(what, _flash_cross(q, kv, lens), q, kv[:, :, 0], kv[:, :, 1], lens):
            failed.append(what)
    qkv = _qkv(2, 272, 48, D, dtype, seed=7)  # 3 query tiles x 48 heads x 2 batches = 288 work items
    what = f"attn_flash many items D={D} {dtype}"
    if not _flash_check(what, _flash_packed(qkv), qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], heads=4):
        failed.append(what)
    T, S = 31, 6
    C = H * D
    x = _qkv(T, S, H, D, dtype, seed=8)  # token-major [T, S, 3, H, D]; a sequence = the T frames of one patch s
    q, k, v = (x[:, :, i].permute(1, 0, 2, 3) for i in range(3))  # [S, T, H, D]
    buf = torch.full((T * S * C + 16,), float("nan"), dtype=dtype, device=DEV)
    out = buf[8:8 + T * S * C]

    def run():
        kernels.attn_flash(x[:, :, 0], x[:, :, 1], x[:, :, 2], S, T, T, H, D, S * 3 * C, 3 * C, S * 3 * C, 3 * C, D**-0.5,
                           out=out, out_row_stride=S * C, out_batch_stride=C)
        return out.clone()
    got = _twice(f"attn_flash strided D={D}", run)
    assert bool(torch.isnan(buf[:8].float()).all() and torch.isnan(buf[-8:].float()).all()), "strided output wrote outside"
    ch = G.flash_chain(q, k, v, D**-0.5)
    what = f"attn_flash strided output D={D} {dtype} T={T} S={S}"
    if not _check(what, got.view(T, S, H, D).permute(1, 0, 2, 3), ch):
        failed.append(what)
    assert not failed, failed


@both
@pytest.mark.parametrize("D", HEAD_DIMS)
def test_attn_flash_exact_index_coded(D, dtype):
    """q = 0: every P is 1 and l the key count, v[b, j, h, d] = [(j + h + b) % D == d], so out = (count of such keys) / l
    -- a dropped, duplicated or wrongly masked key, or a wrong tile, changes a count.  Then a dominant key per row:
    binary-coded keys (+-1 on 12 channels) against q = +-512 times the code of key pi(i), a score gap of 2048 scale log2e
    > 100, so every other P flushes to 0 and out[b, i, h] = v[b, pi(i), h] bit for bit."""
    failed = []
    H = 3
    for nb, nq, nk, lens in ((2, 129, 3600, None), (3, 65, 300, [300, 129, 64]), (1, 1, 1, None)):
        q = torch.zeros(nb, nq, H, D, dtype=dtype, device=DEV)
        k = _hidden(nb, nk, H, D, dtype=dtype, seed=nk)
        j = torch.arange(nk, device=DEV).view(1, nk, 1, 1)
        v = ((j + torch.arange(H, device=DEV).view(1, 1, H, 1) + torch.arange(nb, device=DEV).view(nb, 1, 1, 1)) % D
             == torch.arange(D, device=DEV).view(1, 1, 1, D)).to(dtype)
        kv = torch.stack([k, v], 2)
        what = f"attn_flash q=0 D={D} {dtype} nb={nb} nq={nq} nk={nk} lens={lens}"
        if not _flash_check(what, _flash_cross(q, kv, lens), q, k, v, lens):
            failed.append(what)
        # dominant key
        bits = 12
        code = ((torch.arange(nk, device=DEV).view(nk, 1) >> torch.arange(bits, device=DEV)) & 1).to(torch.float32) * 2 - 1
        kk = torch.zeros(nb, nk, H, D, device=DEV)
        kk[..., :bits] = code.view(1, nk, 1, bits)
        L = lens or [nk] * nb
        pi = [(torch.arange(nq, device=DEV) * 7 + 3 + b) % L[b] for b in range(nb)]
        qq = torch.zeros(nb, nq, H, D, device=DEV)
        for b in range(nb):
            qq[b, :, :, :bits] = 512 * code[pi[b]].view(nq, 1, bits)
        qq, kk = qq.to(dtype), kk.to(dtype)
        vv = _hidden(nb, nk, H, D, dtype=dtype, seed=3)
        kv = torch.stack([kk, vv], 2)
        got = _twice(what, _flash_cross(qq, kv, lens)).view(nb, nq, H, D)
        want = torch.stack([vv[b, pi[b]] for b in range(nb)])
        V.assert_bit_exact(f"attn_flash dominant key D={D} {dtype} nb={nb} nq={nq} nk={nk}", got, want)
    assert not failed, failed


@both
@pytest.mark.parametrize("D", [64, 72, 96, 48])
def test_attn_flash_growing_max_fp64(D, dtype):
    """Scores whose row max grows from key tile to key tile, so every tile rescales O and l."""
    nb, nq, nk, H = 1, 130, 1000, 2
    q = torch.randn(nb, nq, H, D, generator=_gen(1))
    q[..., 0] = 2.0 + q[..., 0].abs()
    k = torch.randn(nb, nk, H, D, generator=_gen(2))
    k[..., 0] += 6.0 * torch.arange(nk).view(1, nk, 1) / nk
    q, k = q.to(dtype).to(DEV), k.to(dtype).to(DEV)
    v = _hidden(nb, nk, H, D, dtype=dtype, seed=3)
    assert _flash_check(f"attn_flash growing max D={D} {dtype}", _flash_cross(q, torch.stack([k, v], 2)), q, k, v)


def _model_rows(n):
    return torch.cat([torch.arange(0, 128), torch.arange(n // 2, n // 2 + 32), torch.arange(n - 128, n)]).to(DEV)


@pytest.mark.parametrize("case", ["opensora-720p-spatial", "opensora-720p-cross", "cogvideox-joint", "osp-v120-3d"])
def test_attn_flash_model_sequences_fp64(case):
    """The models' sequences at full length; the reference on the first, a middle and the last query tile, two heads."""
    failed = []
    if case == "opensora-720p-spatial":  # 720p: 45 x 80 patches = 3600 tokens, 16 heads x 72, two CFG samples
        for dtype in DTYPES:
            qkv = _qkv(2, 3600, 16, 72, dtype, seed=1)
            what = f"attn_flash OpenSora 720p spatial {dtype}"
            if not _flash_check(what, _flash_packed(qkv), qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], rows=_model_rows(3600), heads=2):
                failed.append(what)
    elif case == "opensora-720p-cross":  # 3600 queries against 300 caption keys with caption lengths
        for dtype in DTYPES:
            q = _q(2, 3600, 16, 72, dtype, seed=2)
            kv = _kv(2, 300, 16, 72, dtype, seed=3)
            lens = [300, 37]
            what = f"attn_flash OpenSora 720p cross {dtype}"
            if not _flash_check(what, _flash_cross(q, kv, lens), q, kv[:, :, 0], kv[:, :, 1], lens, rows=_model_rows(3600), heads=2):
                failed.append(what)
    elif case == "cogvideox-joint":  # 226 text + 13 x 30 x 45 video tokens = 17 776, 30 heads x 64, fp16
        qkv = _qkv(1, 17776, 30, 64, torch.float16, seed=4)
        what = "attn_flash CogVideoX joint fp16"
        if not _flash_check(what, _flash_packed(qkv), qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], rows=_model_rows(17776), heads=2):
            failed.append(what)
    else:  # Open-Sora-Plan v1.2.0, 93 x 480p: 24 x 30 x 40 = 28 800 tokens, 24 heads x 96
        for dtype in DTYPES:
            qkv = _qkv(1, 28800, 24, 96, dtype, seed=5)
            what = f"attn_flash Open-Sora-Plan v1.2.0 {dtype}"
            if not _flash_check(what, _flash_packed(qkv), qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], rows=_model_rows(28800), heads=2):
                failed.append(what)
    assert not failed, failed


# =====================================================================================================================
# attn_short
# =====================================================================================================================
def _rope_tables(n, D, seed=4):
    ang = torch.rand(n, D // 2, generator=_gen(seed)) * 6.0
    ang = ang.repeat_interleave(2, 1)
    return torch.cos(ang).to(DEV), torch.sin(ang).to(DEV)


SHORT_N = [1, 2, 15, 16, 17, 20, 31, 32, 33, 48, 63, 64]


@both
@pytest.mark.parametrize("D", [64, 72])
@pytest.mark.parametrize("layout", ["temporal", "spatial"])
def test_attn_short_fp64(layout, D, dtype):
    """flags 0 / 1 / 3 with and without RoPE at every n of SHORT_N (both instantiations); temporal: sequences over the
    frames of each patch of a token-major [B, T, S] buffer; spatial: sequences of n consecutive rows."""
    H = 3
    wq = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=12)
    wk = _rand(D, dtype=dtype, scale=0.2, offset=1.0, seed=13)
    failed = []
    for i, n in enumerate(SHORT_N):
        B, S = 2, 5
        rows = B * n * S
        qkv = _hidden(rows, 3, H, D, dtype=dtype, seed=n)
        if layout == "temporal":
            args = (B, S, n * S, 1, S)
            idx = (torch.arange(B).view(-1, 1, 1) * n * S + torch.arange(S).view(1, -1, 1) + torch.arange(n).view(1, 1, -1) * S)
        else:
            args = (B * S, 1, n, 1, 1)
            idx = torch.arange(rows).view(B * S, 1, n)
        idx = idx.reshape(-1, n).to(DEV)
        for flags in (0, 1, 3):
            for rope in (False, True):
                if (i + flags) % 2 and not rope and n not in (1, 32, 33, 64):
                    continue  # half of the (n, flags) pairs without RoPE
                cos, sin = _rope_tables(n, D) if rope else (None, None)
                what = f"attn_short {layout} D={D} {dtype} n={n} flags={flags} rope={rope}"
                got = _twice(what, lambda: kernels.attn_short(qkv, wq, wk, cos, sin, *args, n, H, D, D**-0.5, flags=flags))
                ch = G.short_chain(qkv[idx.reshape(-1)], wq, wk, cos, sin, n, D**-0.5, flags, dtype)
                if not _check(what, got[idx.reshape(-1)].view(-1, n, H, D), ch):
                    failed.append(what)
    assert not failed, failed


# =====================================================================================================================
# refusals: argument checks that return before any launch
# =====================================================================================================================
def _refused(fn):
    n0 = kernels.launch_count()
    with pytest.raises(VsbError):
        fn()
    assert kernels.launch_count() == n0


@both
def test_gemm_refuses_unaligned_shapes(dtype):
    a, w, bias = _gemm_inputs(16, 64, 12, dtype)
    _refused(lambda: kernels.gemm_bias_act(a, w, bias, 0))  # K % 8
    a, w, bias = _gemm_inputs(16, 12, 64, dtype)
    _refused(lambda: kernels.gemm_bias_act(a, w, bias, 1))  # N % 8
    resid = _hidden(16, 12, dtype=dtype, seed=1)
    _refused(lambda: kernels.gemm_bias_residual(a, w, bias, resid))


@both
def test_attn_flash_refuses(dtype):
    qkv = _qkv(2, 40, 2, 40, dtype, seed=1)
    _refused(_flash_packed(qkv))  # head_dim 40
    q = _hidden(2, 16, 2, 64, dtype=dtype, seed=2)
    kv = _kv(2, 50, 2, 64, dtype, seed=3)
    _refused(_flash_cross(q, kv, [0, 50]))
    _refused(_flash_cross(q, kv, [50, 51]))
    q65 = _hidden(65, 4, 2, 64, dtype=dtype, seed=4)
    kv65 = _kv(65, 8, 2, 64, dtype, seed=5)
    _refused(_flash_cross(q65, kv65, [8] * 65))
    C = 128
    _refused(lambda: kernels.attn_flash(q, kv[:, :, 0], kv[:, :, 1], 2, 16, 50, 2, 64, C + 4, 16 * C, 2 * C, 100 * C, 0.125))


@both
def test_attn_short_refuses(dtype):
    H, D = 2, 64
    qkv = _hidden(2 * 65, 3, H, D, dtype=dtype, seed=1)
    w = _rand(D, dtype=dtype, seed=2)
    _refused(lambda: kernels.attn_short(qkv, w, w, None, None, 2, 1, 65, 1, 1, 65, H, D, 0.125))  # n = 65
    qkv96 = _hidden(2 * 16, 3, H, 96, dtype=dtype, seed=3)
    w96 = _rand(96, dtype=dtype, seed=4)
    _refused(lambda: kernels.attn_short(qkv96, w96, w96, None, None, 2, 1, 16, 1, 1, 16, H, 96, 0.1))  # D = 96
