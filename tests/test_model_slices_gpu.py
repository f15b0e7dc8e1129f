"""The model front ends on the H100 under the sliced parity rule (tests/slice_parity.py): every (sample, frame, 128-row
token tile, 128-column channel tile) of the output within the 16-bit oracle's own error of the fp32 oracle, where the
model tests elsewhere gate one relative L2 over the whole output.

The cases are the real-width ones of those tests, on the same oracles, inputs and golden files.  STDiT3 runs with unequal
caption lengths (the front end's enable_flash_attn caption layout: per-sample key counts from the mask) and with a sample
that has more than one t0 frame.

The negative tests make one small in-bounds change to one kernel wrapper and require the sliced rule to reject the
forward by a margin: a worst slice at least NEGATIVE_MIN_LOAD times its bound, where correct code stays below 0.85.  Each
prints whether the whole-output gate would have passed it.  With these synthetic inputs the t and t0 modulation rows are
independent and every branch is of the order of the residual stream, so a dropped caption token, a flipped frame flag or
an unwritten row tile moves the output by far more than the few per cent a trained model's would, and the whole-output
gate fails them too.  The local change that it does not see is a 128-row tile of one residual branch scaled by 5 %:
asserted to pass the whole-output gate and to fail the sliced rule.

A change spread evenly over a whole sample cannot be sharpened by slicing: it raises every slice of the sample by the same
factor, and the sliced rule sees it only where that factor clears the bound.  The FP8 activation scales of sample 1 at
x 1.02 reach only 1.005 of the bound at 240p, so they run at x 1.04.  One caption token dropped from sample 1's keys is
rejected at the 720p spatial block (2.0 of the bound) but stays below the bound after the 240p block pair (0.93), whose
own 16-bit error is larger; at 240p its load is printed and not asserted."""
import os
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import cases, stdit3_oracle as O, synth
from tests import fp8_rule
from tests.helpers import stdit3_state_dict_template
from tests.slice_parity import assert_sliced_parity, sliced_parity

pytestmark = pytest.mark.gpu
BF, FP16 = torch.bfloat16, torch.float16
DEV = "cuda:0"
NEGATIVE_MIN_LOAD = 1.25


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


# ---- STDiT3 blocks -----------------------------------------------------------------------------------------------------
# name: (B, T, S, L, blocks, hidden, heads, caption lengths, t0 frames per sample)
STDIT3 = {
    "240p": (2, 15, 405, 300, ("spatial", "temporal"), 1152, 16, [300, 173], ([0, 1], [7, 14])),
    "720p": (2, 2, 3600, 300, ("spatial",), 1152, 16, [300, 173], ([0, 1], [1])),
    "T30": (2, 30, 24, 20, ("temporal",), 288, 4, [20, 11], ([0, 1], [29])),
    "T34": (2, 34, 24, 20, ("temporal",), 288, 4, [20, 11], ([0, 1, 2], [17])),
}
CAP = 64  # caption channels


def _oracle_linear(sd, kinds, fp8):
    """F.linear for the oracle; with fp8, the block Linears STDiT3.FP8_LINEARS are the fake-quant Linear of
    tests/fp8_rule.py."""
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3

    names = [".".join(p) for p in STDiT3.FP8_LINEARS]
    quant = {id(sd[f"{k}_blocks.0.{n}.weight"]) for k in kinds for n in names} if fp8 else set()

    def linear(x, w, b=None):
        return fp8_rule.fake_quant_linear(x, w, b).to(x.dtype) if id(w) in quant else F.linear(x, w, b)

    return linear


def _stdit3_oracle(c, fp8):
    """(r16, r32): the caption MLP and the block chain of the oracle in bf16 and in fp32 (varlen cross-attention)."""
    B, T, S, L, kinds, C, H = c["shape"]
    outs = []
    for dt in (BF, torch.float32):
        sd = {k: v.to(dt) for k, v in c["sd"].items()}
        ns = types.SimpleNamespace(**{**{k: getattr(F, k) for k in dir(F) if not k.startswith("_")},
                                      "linear": _oracle_linear(sd, kinds, fp8)})
        x = c["x"].to(dt)
        with pytest.MonkeyPatch.context() as mp, torch.no_grad():
            mp.setattr(O, "F", ns)
            y, y_lens = O.encode_text(sd, c["y"].to(dt), c["mask"], C)
            assert y_lens == c["y_lens"]
            for kind in kinds:
                temporal = kind == "temporal"
                x = O.stdit3_block(sd, f"{kind}_blocks.0.", x, y, c["t"].to(dt), y_lens, c["x_mask"], c["t0"].to(dt), T, S, H,
                                   temporal, sd["rope.freqs"] if temporal else None, cross_varlen=True)
        outs.append(x)
    return outs


def _stdit3_case(store, name, fp8=False):
    """Weights, inputs, the model on the GPU and the two oracles of one case, built once per module."""
    key = (name, fp8)
    if key in store:
        return store[key]
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config

    if fp8:  # the same weights, inputs and model; oracles of their own
        c = dict(_stdit3_case(store, name))
    else:
        B, T, S, L, kinds, C, H, y_lens, t0_frames = STDIT3[name]
        tag = f"slices.{name}."
        cfg = dict(hidden_size=C, num_heads=H, depth=1, caption_channels=CAP, model_max_length=L)
        sd = synth.fill_state_dict(stdit3_state_dict_template(cfg, BF), tag)
        net = STDiT3(STDiT3Config(enable_flash_attn=True, **cfg)).to(BF)
        net.load_state_dict(sd)
        b = cases.block_inputs(BF, C=C, B=B, T=T, S=S, L=L, tag=tag)
        x_mask = torch.ones(B, T, dtype=torch.bool)
        for i, frames in enumerate(t0_frames):
            x_mask[i, frames] = False
        mask = torch.zeros(B, L, dtype=torch.long)
        for i, n in enumerate(y_lens):
            mask[i, :n] = 1
        c = dict(shape=(B, T, S, L, kinds, C, H), sd=sd, net=net.to(DEV).eval(), x=b["x"], t=b["t"], t0=b["t0"], x_mask=x_mask,
                 y=synth.normalish(tag + "cap", (B, 1, L, CAP)).to(BF), mask=mask, y_lens=y_lens)
    c["r16"], c["r32"] = _stdit3_oracle(c, fp8)
    store[key] = c
    return c


@pytest.fixture(scope="module")
def stdit3():
    """case(name, fp8=False) -> the case; the models and oracle outputs are released with the module."""
    store = {}
    yield lambda name, fp8=False: _stdit3_case(store, name, fp8)
    store.clear()
    torch.cuda.empty_cache()


def _stdit3_run(c, fp8=False):
    """The block chain on the kernels, with the caption state (layout and per-sample key counts) that the front end
    derives from y and the mask (STDiT3._text_state)."""
    B, T, S, L, kinds, C, H = c["shape"]
    net = c["net"].set_fp8_linears(fp8)
    try:
        net._text_cache = None
        x = c["x"].to(DEV).clone()
        text = net._text_state(c["y"].to(DEV), c["mask"].to(DEV), B, BF)
        assert text["Lv"] == L and text["kv_lens"] == c["y_lens"]
        t, t0, mask_u8 = c["t"].to(DEV), c["t0"].to(DEV), c["x_mask"].to(torch.uint8).to(DEV)
        with torch.no_grad():
            for kind in kinds:
                x = net._run_block(getattr(net, kind + "_blocks")[0], x, text, t, t0, mask_u8, B, T, S, T, S)
        return x.cpu()
    finally:
        net.set_fp8_linears(False)


def _stdit3_rule(c, got, label, check=True):
    B, T, S, L, kinds, C, H = c["shape"]
    view = lambda v: v.view(B, T, S, C)  # noqa: E731
    fn = assert_sliced_parity if check else sliced_parity
    return fn(label, view(got), view(c["r16"]), view(c["r32"]), "btnc")


@pytest.mark.parametrize("name", list(STDIT3))
def test_stdit3_blocks_sliced(stdit3, name):
    _need_gpu()
    c = stdit3(name)
    _stdit3_rule(c, _stdit3_run(c), f"stdit3 {name} {'+'.join(c['shape'][4])}, captions {c['y_lens']}")


@pytest.mark.parametrize("name", ["240p", "720p"])
def test_stdit3_fp8_blocks_sliced(stdit3, name):
    """FP8 mode (qkv and fc1 on the e4m3 GEMM) against the oracle whose qkv and fc1 are the fake-quant Linear."""
    _need_gpu()
    c = stdit3(name, fp8=True)
    _stdit3_rule(c, _stdit3_run(c, fp8=True), f"stdit3 fp8 {name}")


# ---- negative tests: one small in-bounds change to one kernel wrapper -----------------------------------------------------
def _drop_last_caption_token(K, mp):
    f = K.attn_flash

    def attn_flash(*a, kv_lens=None, **kw):
        if kv_lens is not None:
            kv_lens = list(kv_lens)
            kv_lens[1] -= 1
        return f(*a, kv_lens=kv_lens, **kw)

    mp.setattr(K, "attn_flash", attn_flash)


def _flip_one_frame_flag(K, mp):
    """Sample 1's frame 0 (a t frame in every case) takes the t0 modulation rows in the LayerNorm-modulate passes."""
    f = K.ln_modulate

    def ln_modulate(x, mod, x_mask_u8, *a, **kw):
        if x_mask_u8 is not None:
            x_mask_u8 = x_mask_u8.clone()
            x_mask_u8[1, 0] ^= 1
        return f(x, mod, x_mask_u8, *a, **kw)

    mp.setattr(K, "ln_modulate", ln_modulate)


def _last_row_tile(K, mp, branch_scale):
    """The first residual GEMM of the chain writes resid + branch_scale * branch in its last 128-row tile (the end of
    sample 1): 0 leaves the tile unwritten."""
    f = K.gemm_bias_residual
    calls = []

    def gemm_bias_residual(a, w, bias, resid, *args, **kw):
        M = a.numel() // a.shape[-1]
        rows = slice((M - 1) // 128 * 128, M)
        keep = resid.view(M, -1)[rows].clone() if not calls else None
        out = f(a, w, bias, resid, *args, **kw)
        if keep is not None:
            tile = out.view(M, -1)[rows]
            tile.copy_(keep.float() + branch_scale * (tile.float() - keep.float()))
        calls.append(M)
        return out

    mp.setattr(K, "gemm_bias_residual", gemm_bias_residual)


def _scale_sample1_fp8_activations(K, mp):
    f = K.gemm_fp8_bias_act

    def gemm_fp8_bias_act(a, a_scale, *args, **kw):
        a_scale = a_scale.clone()
        rows = a_scale.view(-1)
        rows[rows.numel() // 2:] *= 1.04
        return f(a, a_scale, *args, **kw)

    mp.setattr(K, "gemm_fp8_bias_act", gemm_fp8_bias_act)


# id: (change, patch, FP8 mode, whether the whole-output gate must pass it, the cases where the rejection is asserted)
BOTH = ("240p", "720p")
NEGATIVE = {
    "kv_lens": ("cross-attention kv_lens[1] - 1", _drop_last_caption_token, False, False, ("720p",)),
    "x_mask": ("ln_modulate x_mask flag of sample 1 frame 0 flipped", _flip_one_frame_flag, False, False, BOTH),
    "tile_unwritten": ("gemm_bias_residual last row tile of sample 1 unwritten", lambda K, mp: _last_row_tile(K, mp, 0.0),
                       False, False, BOTH),
    "tile_branch_x1.05": ("gemm_bias_residual branch of the last row tile of sample 1 x 1.05",
                          lambda K, mp: _last_row_tile(K, mp, 1.05), False, True, BOTH),
    "fp8_scale_x1.04": ("fp8 GEMM activation scales of sample 1 x 1.04", _scale_sample1_fp8_activations, True, False, BOTH),
}


@pytest.mark.parametrize("name", ["240p", "720p"])
@pytest.mark.parametrize("neg", list(NEGATIVE))
def test_stdit3_negative_rejected(stdit3, name, neg):
    _need_gpu()
    from videosys_b200 import kernels as K

    change, patch, fp8, below_old_gate, asserted_at = NEGATIVE[neg]
    c = stdit3(name, fp8=fp8)
    with pytest.MonkeyPatch.context() as mp:
        patch(K, mp)
        got = _stdit3_run(c, fp8=fp8)
    rep = _stdit3_rule(c, got, f"NEGATIVE stdit3 {'fp8 ' if fp8 else ''}{name}: {change}", check=False)
    print(rep.describe())
    if name not in asserted_at:
        print(f"[slices] {change} at {name}: spread evenly over sample 1 and below the rule's resolution there; load reported, "
              f"not asserted")
        return
    assert rep.worst >= NEGATIVE_MIN_LOAD, f"{change}: worst slice only {rep.worst:.3f}x its bound"
    if below_old_gate:
        assert rep.old_gate_ok, f"{change}: meant as a change the whole-output gate does not see ({rep.whole_ratio:.3f})"


# ---- CogVideoX ---------------------------------------------------------------------------------------------------------
def _cogx_fill(net, tag):
    from tests.test_cogvideox_gpu import _fill

    sd = _fill(net)
    for k in sd:
        if k.endswith("norm_final.weight") or k.endswith("norm_out.norm.weight"):
            sd[k] = (1.0 + 0.2 * synth.uniform(tag + k, tuple(sd[k].shape))).to(sd[k].dtype)
    return sd


def test_cogvideox_2b_block_fp16_sliced():
    """The 2b width (30 heads x 64) in its fp16: the video stream as 3 frames of 15 x 30 patches, and the text stream."""
    _need_gpu()
    from oracle import cogvideox_oracle as CO
    from videosys_b200.models.transformers.cogvideox_transformer_3d import CogVideoXBlockStack

    dt, heads, D, B, Fr, P, Nt = FP16, 30, 64, 2, 3, 450, 226
    C = heads * D
    net = CogVideoXBlockStack(heads, D, 1, 512).to(dt)
    sd = _cogx_fill(net, "slices.cogx.")
    net.load_state_dict(sd)
    net = net.to(DEV).eval()
    hid = synth.normalish("slices.cogx.h", (B, Fr * P, C)).to(dt)
    enc = synth.normalish("slices.cogx.e", (B, Nt, C)).to(dt)
    temb = synth.normalish("slices.cogx.t", (B, 512)).to(dt)
    oh, oe = (v.cpu() for v in net(hid.to(DEV), enc.to(DEV), temb.to(DEV)))
    with torch.no_grad():
        h16, e16 = CO.block(sd, "transformer_blocks.0.", hid, enc, temb, heads)
        sd32 = {k: v.float() for k, v in sd.items()}
        h32, e32 = CO.block(sd32, "transformer_blocks.0.", hid.float(), enc.float(), temb.float(), heads)
    v = lambda t: t.view(B, Fr, P, C)  # noqa: E731
    assert_sliced_parity("cogvideox 2b fp16 video", v(oh), v(h16), v(h32), "btnc")
    assert_sliced_parity("cogvideox 2b fp16 text", oe, e16, e32, "bnc")


def test_cogvideox_5b_rotary_forward_bf16_sliced():
    """The 5b layout (48 heads x 64, 3-D rotary tables, 4096-wide text) in its bf16: the transformer forward, one layer."""
    _need_gpu()
    from oracle import cogvideox_oracle as CO
    from tests.test_cogvideox_gpu import SMALL, SMALL_O
    from videosys_b200.models.transformers.cogvideox_transformer_3d import CogVideoXTransformer3DModel

    dt = BF
    cfg = dict(SMALL, num_attention_heads=48, text_embed_dim=4096, time_embed_dim=512, num_layers=1,
               use_rotary_positional_embeddings=True)
    ocfg = dict(SMALL_O, heads=48, layers=1)
    net = CogVideoXTransformer3DModel(**cfg).to(dt)
    sd = _cogx_fill(net, "slices.cogx5b.")
    net.load_state_dict(sd)
    net = net.to(DEV).eval()
    B, Fr, H, W = 2, 3, 12, 16
    lat = synth.normalish("slices.cogx5b.lat", (B, Fr, 4, H, W)).to(dt)
    txt = synth.normalish("slices.cogx5b.txt", (B, 16, 4096)).to(dt)
    ts = torch.tensor([499, 499], dtype=torch.int64)
    rot = CO.rotary_3d(64, CO.resize_crop_region_for_grid((6, 8), 45, 30), (6, 8), Fr)
    out = net(lat.to(DEV), txt.to(DEV), ts.to(DEV), image_rotary_emb=(rot[0].to(DEV), rot[1].to(DEV)), return_dict=False)[0].cpu()
    with torch.no_grad():
        r16 = CO.transformer_forward(sd, ocfg, lat, txt, ts, rotary=rot)
        r32 = CO.transformer_forward({k: v.float() for k, v in sd.items()}, ocfg, lat.float(), txt.float(), ts, rotary=rot)
    assert_sliced_parity("cogvideox 5b rotary bf16", out, r16, r32, "btcnn")


# ---- Latte -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [FP16, BF], ids=["fp16", "bf16"])
def test_latte_config1_forward_sliced(dt):
    """BASELINE config 1: latent [2, 4, 16, 32, 32], 120 text tokens, hidden 1152 = 16 heads x 72, 2 of the 28 layers."""
    _need_gpu()
    from oracle import latte_oracle as LO
    from videosys_b200.models.transformers.latte_transformer_3d import LatteT2V

    cfg = dict(num_layers=2, sample_size=32, caption_channels=4096, video_length=16)
    ocfg = dict(heads=16, head_dim=72, layers=2, patch=2, sample_size=32, out_channels=8, video_length=16)
    shape, L = (2, 4, 16, 32, 32), 120
    net = LatteT2V(**cfg).to(dt)
    sd = synth.fill_state_dict(net.state_dict(), "lattef.")
    net.load_state_dict(sd)
    net = net.to(DEV).eval()
    lat = synth.normalish("lattef.lat", shape).to(dt)
    txt = synth.normalish("lattef.txt", (shape[0], L, 4096)).to(dt)
    ts = torch.tensor([999] * shape[0], dtype=torch.int64)
    out = net(lat.to(DEV), timestep=ts.to(DEV), encoder_hidden_states=txt.to(DEV), return_dict=False)[0].cpu()
    with torch.no_grad():
        r16 = LO.transformer_forward(sd, ocfg, lat, ts, txt)
        r32 = LO.transformer_forward({k: v.float() for k, v in sd.items()}, ocfg, lat.float(), ts, txt.float())
    assert_sliced_parity(f"latte config 1 {dt}", out, r16, r32, "bctnn")


# ---- Vchitect ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [BF, FP16], ids=["bf16", "fp16"])
def test_vchitect_wide_forward_sliced(dt):
    """Vchitect-2.0-2B's width, 2 of its 24 layers, 8 frames of 288 x 480, 77 + 256 text tokens."""
    _need_gpu()
    from oracle import vchitect_oracle as VO
    from tests.test_vchitect_gpu import WIDE, WIDE_O, _net

    shape, L = (1, 8, 16, 36, 60), 333
    net, sd = _net(WIDE, dt, "vchf.")
    lat = synth.normalish("vchf.lat", shape).to(dt)
    enc = synth.normalish("vchf.enc", (1, L, WIDE["joint_attention_dim"])).to(dt)
    pooled = synth.normalish("vchf.pool", (1, WIDE["pooled_projection_dim"])).to(dt)
    ts = torch.tensor([500.0])
    out = net(lat.cuda(), enc.cuda(), pooled.cuda(), ts.cuda(), return_dict=False)[0].cpu()
    with torch.no_grad():
        r16 = VO.transformer_forward(sd, WIDE_O, lat, enc, pooled, ts)
        r32 = VO.transformer_forward({k: v.float() for k, v in sd.items()}, WIDE_O, lat.float(), enc.float(), pooled.float(), ts)
    assert_sliced_parity(f"vchitect wide {dt}", out, r16, r32, "tcnn")  # batch 1: [frames, channels, H, W]


# ---- Open-Sora-Plan ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt,dn", [(BF, "bf16"), (FP16, "fp16")], ids=["bf16", "fp16"])
def test_osp_v110_wide_vs_reference_golden_sliced(golden_dir, dt, dn):
    """The released v1.1.0 width against the reference's own outputs; the golden file holds a seeded sample of them."""
    _need_gpu()
    from oracle import osp_cases as OC
    from tests.test_osp_gpu import _net

    gold = torch.load(os.path.join(golden_dir, "osp_v110.pt"))
    name = "wide_rope"
    net = _net(name, dt)
    x, enc, m, tt = OC.inputs(name, dt)
    out = net(x.cuda(), timestep=tt.cuda(), all_timesteps=[900, 500], encoder_hidden_states=enc.cuda(),
              attention_mask=torch.ones(x.shape[0], x.shape[2], x.shape[3], x.shape[4]), encoder_attention_mask=m,
              return_dict=False)[0].cpu()
    shape, idx = gold[f"{name}.shape"], gold[f"{name}.idx"]
    assert list(out.shape) == shape
    assert_sliced_parity(f"osp v110 {name} {dn}", out.flatten()[idx.long()], gold[f"{name}.{dn}"], gold[f"{name}.fp32"], "bctnn",
                         idx=idx, shape=shape)


@pytest.mark.parametrize("dt,dn", [(BF, "bf16"), (FP16, "fp16")], ids=["bf16", "fp16"])
def test_osp_v120_wide_vs_reference_golden_sliced(golden_dir, dt, dn):
    _need_gpu()
    from oracle import osp_cases as OC
    from tests.test_osp_gpu import _net12

    gold = torch.load(os.path.join(golden_dir, "osp_v120.pt"))
    name = "wide_rope"
    net = _net12(name, dt)
    x, enc, m, tt = OC.inputs12(name, dt)
    out = net(x.cuda(), timestep=tt.cuda(), encoder_hidden_states=enc.cuda(), encoder_attention_mask=m, return_dict=False)[0].cpu()
    assert_sliced_parity(f"osp v120 {name} {dn}", out, gold[f"{name}.{dn}"], gold[f"{name}.fp32"], "bctnn")
