"""Pins the oracle and the product front ends by EXECUTING THE UNMODIFIED REFERENCE where its checkout is available
(``VSB_REFERENCE_ROOT``), and against its stored results everywhere else.

Every comparison takes the reference side through ``_ref(key, fn)``: with the checkout present fn() runs the reference (and,
with VSB_RECORD_GOLDEN=1, stores its result under tests/golden/reference/, one file per key prefix); without it the stored
result is used.  Tensors above 16384 elements are stored as a fixed seeded sample of 4096 elements with their indices
(``_pair`` applies the same sample to the value under test); module weights as state-dict templates (key / shape / dtype)
that synth.fill_state_dict fills deterministically."""
import os
import threading

import pytest
import torch

from oracle import cases, dsp_oracle, pab_oracle, ref_loader, stdit3_oracle as O, synth

_GOLD_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")
_gold_cache = {}
_SAMPLE_OVER, _SAMPLE_N = 16384, 4096


def _pack(v):
    if torch.is_tensor(v) and v.numel() > _SAMPLE_OVER:
        idx = torch.randperm(v.numel(), generator=torch.Generator().manual_seed(0))[:_SAMPLE_N].sort().values
        return {"sampled_shape": list(v.shape), "idx": idx.to(torch.int32), "vals": v.flatten()[idx].clone()}
    if isinstance(v, (list, tuple)):
        return type(v)(_pack(x) for x in v)
    if isinstance(v, dict):
        return v if v.get("__template__") else {k: _pack(x) for k, x in v.items()}  # templates are stored whole
    return v


def _pair(got, want):
    """(got, want) as compared: a stored sample of want selects the same elements of got."""
    if isinstance(want, dict) and "sampled_shape" in want:
        assert list(got.shape) == want["sampled_shape"], (tuple(got.shape), want["sampled_shape"])
        return got.flatten()[want["idx"].long()], want["vals"]
    assert got.shape == want.shape, (tuple(got.shape), tuple(want.shape))
    return got, want


def _assert_same(got, want, dtype):
    """Bit for bit against the reference.  A stored 16-bit reference result was produced by the CPU kernels of the host that
    recorded it, and torch's 16-bit CPU matmuls accumulate in an order that depends on the instruction set; replayed on
    another host, results computed in 16 bits (`dtype`) are held to the 16-bit rounding level instead (fp32 stays bit for bit)."""
    g, w = _pair(got, want)
    if ref_loader.available() or dtype == torch.float32:
        assert torch.equal(g, w), (g.double() - w.double()).abs().max()
        return
    rel = ((g.double() - w.double()).norm() / w.double().norm()).item()
    assert g.dtype == w.dtype and rel <= (1e-2 if dtype == torch.bfloat16 else 2e-3), rel


def _ref(key, fn):
    """The reference's result for ``key``: fn() where the reference checkout is present (stored when VSB_RECORD_GOLDEN=1),
    the stored result elsewhere."""
    path = os.path.join(_GOLD_DIR, key.split(".")[0] + ".pt")
    if ref_loader.available() and fn is not None:
        val = fn()
        if os.environ.get("VSB_RECORD_GOLDEN") == "1":
            os.makedirs(_GOLD_DIR, exist_ok=True)
            d = torch.load(path) if os.path.exists(path) else {}
            d[key] = _pack(val)
            torch.save(d, path)
        return val
    if path not in _gold_cache:
        _gold_cache[path] = torch.load(path)
    assert key in _gold_cache[path], f"{key} missing from {path}"
    return _gold_cache[path][key]


def _template(sd, keep=()):
    """Key / shape / dtype of a reference module's state_dict (what synth.fill_state_dict needs); `keep` = entries whose
    values are not weights (tables) and are stored as they are."""
    keep_value = lambda k: k in keep or k.endswith("rope.freqs") or k.endswith("inv_freq")  # noqa: E731  (copied by fill_state_dict)
    t = {k: (list(v.shape), str(v.dtype)) if torch.is_floating_point(v) and not keep_value(k) else v.clone() for k, v in sd.items()}
    t["__template__"] = True
    return t


def _from_template(t):
    return {k: torch.zeros(v[0], dtype=getattr(torch, v[1].split(".")[-1])) if isinstance(v, tuple) else v for k, v in t.items()
            if k != "__template__"}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_forward_bit_exact(dtype):
    c = cases.small_model_cfg(depth=2)
    inp = cases.forward_inputs(dtype)

    def reference():
        net = ref_loader.build_stdit3(dtype=dtype, **c)
        net.load_state_dict(synth.fill_state_dict(net.state_dict(), "vsref."))
        with torch.no_grad():
            return _template(net.state_dict()), net(inp["x"], inp["timestep"], inp["y"], mask=inp["mask"], x_mask=inp["x_mask"],
                                                    fps=inp["fps"], height=inp["height"], width=inp["width"])

    tmpl, ref = _ref(f"stdit3_fwd.{dtype}", reference)
    sd = synth.fill_state_dict(_from_template(tmpl), "vsref.")
    with torch.no_grad():
        out = O.stdit3_forward(sd, cases.oracle_cfg(c), **inp)
    _assert_same(out, ref, dtype)


def test_forward_with_pab_bit_exact_over_steps():
    """PAB on (attn + cross broadcast; mlp_broadcast=False, the only mode the reference can run for
    OpenSora, SURVEY fact 7): reuse-by-reference semantics and counters over 8 consecutive steps."""
    dtype = torch.bfloat16
    c = cases.small_model_cfg(depth=2)
    steps = [1000, 900, 860, 800, 700, 600, 500, 300]

    def step_inputs(i, t):
        inp = cases.forward_inputs(dtype)
        inp["x"] = synth.normalish(f"pab.x{i}", tuple(inp["x"].shape))
        inp["timestep"] = torch.tensor([float(t)] * 2)
        return inp

    def reference():
        P = ref_loader.load().pab_mgr
        net = ref_loader.build_stdit3(dtype=dtype, **c)
        net.load_state_dict(synth.fill_state_dict(net.state_dict(), "vsref."))
        P.set_pab_manager(P.PABConfig(spatial_broadcast=True, spatial_threshold=[450, 930], spatial_range=2,
                                      temporal_broadcast=True, temporal_threshold=[450, 930], temporal_range=4,
                                      cross_broadcast=True, cross_threshold=[450, 930], cross_range=6))
        P.update_steps(len(steps))
        outs = []
        try:
            with torch.no_grad():
                for i, t in enumerate(steps):
                    inp = step_inputs(i, t)
                    outs.append(net(inp["x"], inp["timestep"], inp["y"], mask=inp["mask"], x_mask=inp["x_mask"], fps=inp["fps"],
                                    height=inp["height"], width=inp["width"]))
        finally:
            P.PAB_MANAGER = None
        return _template(net.state_dict()), outs

    tmpl, refs = _ref("stdit3_pab.steps", reference)
    sd = synth.fill_state_dict(_from_template(tmpl), "vsref.")
    gate = pab_oracle.opensora_default(len(steps))
    states = {k: [O.BlockPABState() for _ in range(2)] for k in ("spatial", "temporal")}
    with torch.no_grad():
        for i, t in enumerate(steps):
            o = O.stdit3_forward(sd, cases.oracle_cfg(c), pab=gate, pab_states=states, **step_inputs(i, t))
            _assert_same(o, refs[i], dtype)


def test_pab_gate_matches_reference_manager():
    import random

    rnd = random.Random(0)
    scenarios = []  # (PABConfig kwargs, oracle spec, steps, timesteps queried per gate)
    for _ in range(20):
        kw, spec = {}, {}
        for k in ("spatial", "temporal", "cross"):
            on = rnd.random() < 0.7
            lo = rnd.randrange(0, 600)
            hi = lo + rnd.randrange(1, 500)
            rg = rnd.randrange(1, 7)
            kw.update({f"{k}_broadcast": on, f"{k}_threshold": [lo, hi], f"{k}_range": rg})
            spec[k] = (on, (lo, hi), rg)
        steps = rnd.randrange(1, 40)
        queries = {k: [rnd.choice([None, rnd.randrange(0, 1100)]) for _ in range(3 * steps)] for k in ("spatial", "temporal", "cross")}
        scenarios.append((kw, spec, steps, queries))

    def reference():
        P = ref_loader.load().pab_mgr
        res = []
        try:
            for kw, _, steps, queries in scenarios:
                P.set_pab_manager(P.PABConfig(**kw))
                P.update_steps(steps)
                for k, fn in (("spatial", P.if_broadcast_spatial), ("temporal", P.if_broadcast_temporal), ("cross", P.if_broadcast_cross)):
                    c = 0
                    for t in queries[k]:
                        f, c = fn(t, c)
                        res.append((bool(f), int(c)))
        finally:
            P.PAB_MANAGER = None
        return res

    want = _ref("pab_gate.scenarios", reference)
    got = []
    for _, spec, steps, queries in scenarios:
        g = pab_oracle.PABGate(steps=steps, **spec)
        for k in ("spatial", "temporal", "cross"):
            c = 0
            for t in queries[k]:
                f, c = g.gate(k, t, c)
                got.append((bool(f), int(c)))
    assert [tuple(x) for x in want] == got


class _FakeDist:
    """Thread-per-rank stand-in for torch.distributed so the reference comm functions run on CPU."""

    def __init__(self, sp):
        self.sp = sp
        self.board = [None] * sp
        self.bar = threading.Barrier(sp)
        self.local = threading.local()
        self.ProcessGroup = object

    def get_world_size(self, group=None):
        return self.sp

    def get_rank(self, group=None):
        return self.local.rank

    def all_to_all(self, output_list, input_list, group=None):
        r = self.local.rank
        self.board[r] = input_list
        self.bar.wait()
        for src in range(self.sp):
            output_list[src].copy_(self.board[src][r])
        self.bar.wait()


def _run_ranks(sp, fn):
    fake = _FakeDist(sp)
    comm = ref_loader.load().comm
    old = comm.dist
    comm.dist = fake
    outs, errs = [None] * sp, []

    def body(r):
        fake.local.rank = r
        try:
            outs[r] = fn(comm, r)
        except Exception as e:  # pragma: no cover
            errs.append(e)
            fake.bar.abort()

    try:
        th = [threading.Thread(target=body, args=(r,)) for r in range(sp)]
        [t.start() for t in th]
        [t.join() for t in th]
    finally:
        comm.dist = old
    assert not errs, errs
    return outs


@pytest.mark.parametrize("sp,T,S", [(2, 5, 9), (4, 5, 9), (8, 20, 24), (4, 4, 8), (2, 15, 405)])
def test_dsp_reshard_matches_reference_comm(sp, T, S):
    B, C = 2, 16
    full = synth.normalish(f"dsp{sp}{T}{S}", (B, T, S, C))
    tp, spd = dsp_oracle.pad_amount(T, sp), dsp_oracle.pad_amount(S, sp)
    res = dsp_oracle.split_sequence(full, sp, dim=2)

    def fn(comm, r):
        x = comm._split_sequence_func(full, None, 2, spd)
        a = comm.all_to_all_with_pad(x, None, scatter_dim=1, gather_dim=2, scatter_pad=tp, gather_pad=spd)
        b = comm.all_to_all_with_pad(a, None, scatter_dim=2, gather_dim=1, scatter_pad=spd, gather_pad=tp)
        return x, a, b

    # the reshard only moves token vectors: the reference runs on 1-channel position ids (0 = padding) and the stored
    # permutation is applied to `full`, which keeps the golden file small
    ids = torch.arange(1, B * T * S + 1, dtype=torch.float64).reshape(B, T, S, 1)

    def fn_ids(comm, r):
        x = comm._split_sequence_func(ids, None, 2, spd)
        a = comm.all_to_all_with_pad(x, None, scatter_dim=1, gather_dim=2, scatter_pad=tp, gather_pad=spd)
        b = comm.all_to_all_with_pad(a, None, scatter_dim=2, gather_dim=1, scatter_pad=spd, gather_pad=tp)
        return tuple(o[..., 0].to(torch.int32) for o in (x, a, b))

    table = torch.cat([torch.zeros(1, C), full.reshape(-1, C)])
    outs = [tuple(table[o.long()] for o in rank) for rank in _ref(f"dsp.{sp}.{T}.{S}", lambda: _run_ranks(sp, fn_ids))]
    if ref_loader.available():  # the permutation reproduces the reference on the real data
        for got, want in zip(_run_ranks(sp, fn), outs):
            assert all(torch.equal(g, w) for g, w in zip(got, want))
    parts = [p.reshape(B, -1, C) for p in res]
    sw, new_s, new_t = dsp_oracle.dynamic_switch(parts, T, S, to_spatial_shard=False)
    back, s2, t2 = dsp_oracle.dynamic_switch(sw, T, S, to_spatial_shard=True)
    padded_t = torch.cat([full, torch.zeros(B, tp, S, C)], 1)
    for r in range(sp):
        x, a, b = outs[r]
        assert torch.equal(x, res[r])
        assert torch.equal(a.reshape(B, -1, C), sw[r]) and (a.shape[1], a.shape[2]) == (new_t, new_s)
        assert torch.equal(a, padded_t[:, r * new_t:(r + 1) * new_t])  # Appendix E: a slice of the T-padded tensor
        assert torch.equal(b.reshape(B, -1, C), back[r]) and torch.equal(b, x)
    assert torch.equal(dsp_oracle.gather_sequence([o[2] for o in outs], 2, spd), full)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_cogvideox_layernorm_zero(dtype):
    """The in-tree half of the CogVideoX block: CogVideoXLayerNormZero (models/modules/normalization.py:36-57)."""
    from oracle import cogvideox_oracle as CO

    h = synth.normalish("lnz.h", (2, 9, 128)).to(dtype)
    e = synth.normalish("lnz.e", (2, 4, 128)).to(dtype)
    t = synth.normalish("lnz.t", (2, 64)).to(dtype)

    def weights(template):
        sd = {"n." + k: v for k, v in synth.fill_state_dict(template, "lnz.").items()}
        sd["n.norm.weight"] = (1 + 0.2 * synth.uniform("lnz.w", (128,))).to(dtype)
        return sd

    def reference():
        N = ref_loader.load().normalization
        mod = N.CogVideoXLayerNormZero(64, 128, True, 1e-5, bias=True).to(dtype)
        mod.load_state_dict({k[2:]: v for k, v in weights(mod.state_dict()).items()})
        with torch.no_grad():
            return _template(mod.state_dict()), mod(h, e, t)

    tmpl, ref = _ref(f"lnz.{dtype}", reference)
    sd = weights(_from_template(tmpl))
    with torch.no_grad():
        got = CO.layer_norm_zero(sd, "n.", h, e, t)
    for a, b in zip(ref, got):
        assert torch.equal(a, b)


def test_cogvideox_ddim_scheduler_vs_reference():
    """videosys_b200's CogVideoXDDIMScheduler against the reference's own class (executed unmodified): trailing timesteps,
    the SNR-shifted / zero-terminal-SNR alphas, and 50 v-prediction steps on random tensors."""
    from videosys_b200.schedulers.scheduling_ddim_cogvideox import CogVideoXDDIMScheduler as Ours

    kw = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
              set_alpha_to_one=True, steps_offset=0, prediction_type="v_prediction", timestep_spacing="trailing",
              rescale_betas_zero_snr=True, snr_shift_scale=3.0)

    def steps(sched, call):
        g = torch.Generator().manual_seed(0)
        x = torch.randn(1, 3, 4, 6, 6, generator=g)
        outs = []
        for t in sched.timesteps:
            x = call(sched, torch.randn(x.shape, generator=g), t, x)
            outs.append(x)
        return torch.stack(outs)

    def reference():
        ref = ref_loader.load_cogvideox_scheduler()(**kw)
        ts = {}
        for n in (50, 30, 7):
            ref.set_timesteps(n)
            ts[n] = ref.timesteps.tolist()
        ref.set_timesteps(50)
        return ref.alphas_cumprod, ts, list(steps(ref, lambda s, v, t, x: s.step(v, t, x, return_dict=False)[0]).unbind(0))

    alphas, ts, xr = _ref("cogx_ddim", reference)
    ours = Ours(**kw)
    assert torch.equal(alphas, ours.alphas_cumprod)
    for n in (50, 30, 7):
        ours.set_timesteps(n)
        assert ts[n] == ours.timesteps.tolist()
    ours.set_timesteps(50)
    xo = steps(ours, lambda s, v, t, x: s.step(v, int(t), x)[0])
    for i, t in enumerate(ts[50]):
        assert torch.allclose(xr[i].float(), xo[i].float(), rtol=1e-5, atol=1e-6), t


def _vchitect_ref_attention(C, H, context_pre_only, dtype):
    A = ref_loader.load().attentions
    attn = A.VchitectAttention(query_dim=C, cross_attention_dim=None, added_kv_proj_dim=C, dim_head=C // H, heads=H,
                               out_dim=C, context_pre_only=context_pre_only, bias=True, processor=A.VchitectAttnProcessor())
    attn = attn.to(dtype).eval()
    attn.parallel_manager = ref_loader.SingleRankPM()
    sd = synth.fill_state_dict(attn.state_dict(), "vchattn.")
    attn.load_state_dict(sd)
    return attn, {"a." + k: v for k, v in sd.items()}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("Fr,S,L,pre_only", [(5, 12, 7, False), (5, 12, 7, True), (1, 12, 7, False)])
def test_vchitect_attention_vs_reference(Fr, S, L, pre_only, dtype):
    """oracle/vchitect_oracle.attention against the reference's own VchitectAttention + VchitectAttnProcessor
    (models/modules/attentions.py:321-949, executed unmodified): temporal (RoPE), cross (frame-0 text keys) and spatial
    joint attention, the 1.1 mix, the output projections of both streams; bit for bit."""
    from oracle import vchitect_oracle as VO

    C, H = 64, 4
    nh = synth.normalish("vch.h", (Fr, S, C)).to(dtype)
    ne = synth.normalish("vch.e", (Fr, L, C)).to(dtype)
    fc = VO.freqs_cis(C // H, 64, theta=1e6)

    def reference():
        attn, sd = _vchitect_ref_attention(C, H, pre_only, dtype)
        with torch.no_grad():
            rv, re = attn(hidden_states=nh, encoder_hidden_states=ne, freqs_cis=fc, full_seqlen=Fr, Frame=Fr,
                          timestep=torch.tensor([500]))
        return _template(attn.state_dict()), rv, re

    tmpl, rv, re = _ref(f"vch_attn.{Fr}.{S}.{L}.{pre_only}.{dtype}", reference)
    sd = {"a." + k: v for k, v in synth.fill_state_dict(_from_template(tmpl), "vchattn.").items()}
    with torch.no_grad():
        ov, oe = VO.attention(sd, "a.", nh, ne, fc, H, Fr, pre_only)
    assert torch.equal(rv, ov)
    assert torch.equal(re, oe)


def test_vchitect_attention_pab_vs_reference():
    """The three PAB gates of the processor (:838-895: temporal, cross, spatial, in this order) over 8 steps."""
    from oracle import vchitect_oracle as VO

    C, H, Fr, S, L = 64, 4, 4, 10, 6
    ts = [900, 700, 650, 600, 550, 500, 450, 50]
    fc = VO.freqs_cis(C // H, 64, theta=1e6)
    inputs = [(synth.normalish(f"vchp.h{step}", (Fr, S, C)), synth.normalish(f"vchp.e{step}", (Fr, L, C))) for step in range(len(ts))]

    def reference():
        P = ref_loader.load().pab_mgr
        attn, _ = _vchitect_ref_attention(C, H, False, torch.float32)
        P.set_pab_manager(P.PABConfig(spatial_broadcast=True, spatial_threshold=[100, 800], spatial_range=2, temporal_broadcast=True,
                                      temporal_threshold=[100, 800], temporal_range=3, cross_broadcast=True,
                                      cross_threshold=[100, 800], cross_range=4))
        P.update_steps(8)
        outs = []
        try:
            with torch.no_grad():
                for (nh, ne), t in zip(inputs, ts):
                    outs.append(attn(hidden_states=nh, encoder_hidden_states=ne, freqs_cis=fc, full_seqlen=Fr, Frame=Fr,
                                     timestep=torch.tensor([t])))
        finally:
            P.PAB_MANAGER = None
        return _template(attn.state_dict()), outs

    tmpl, refs = _ref("vch_attn_pab.steps", reference)
    sd = {"a." + k: v for k, v in synth.fill_state_dict(_from_template(tmpl), "vchattn.").items()}
    counts = {"spatial": 0, "temporal": 0, "cross": 0}
    cache = {}
    G = pab_oracle.PABGate((True, (100, 800), 2), (True, (100, 800), 3), (True, (100, 800), 4), 8)
    for step, ((nh, ne), t) in enumerate(zip(inputs, ts)):
        def gate(kind, t=t):
            hit, counts[kind] = G.gate(kind, t, counts[kind])
            return hit

        with torch.no_grad():
            ov, oe = VO.attention(sd, "a.", nh, ne, fc, H, Fr, False, gate, cache)
        rv, re = refs[step]
        assert torch.equal(*_pair(ov, rv)) and torch.equal(*_pair(oe, re)), step


# ---- Open-Sora-Plan v1.1.0: the product's host logic against the UNMODIFIED reference model --------------------------------
OSP_SMALL = dict(num_attention_heads=2, attention_head_dim=72, in_channels=4, out_channels=8, num_layers=2,
                 cross_attention_dim=144, attention_bias=True, sample_size=(8, 8), patch_size=2, activation_fn="gelu-approximate",
                 norm_type="ada_norm_single", norm_elementwise_affine=False, norm_eps=1e-6, caption_channels=32, video_length=5,
                 attention_mode="math", use_rope=True)


def _osp_ref(cfg, tag="osp."):
    ref = ref_loader.build_osp_v110(**cfg)
    ref.load_state_dict(synth.fill_state_dict(ref.state_dict(), tag))
    return ref


def _osp_net(cfg, tmpl, tag="osp."):
    from videosys_b200.models.transformers.open_sora_plan_v110_transformer_3d import LatteT2V

    net = LatteT2V(**cfg)
    net.load_state_dict(synth.fill_state_dict(_from_template(tmpl), tag))  # strict: same parameter / buffer names as the reference
    return net.eval()


def _osp_inputs(B, Fr, HW, L=7, tag="osp."):
    x = synth.normalish(tag + "x", (B, 4, Fr, *HW))
    enc = synth.normalish(tag + "enc", (B, 1, L, 32))
    m = torch.ones(B, 1, L)
    m[B - 1, 0, L - 2:] = 0  # tokenizer padding on the last sample
    return x, enc, m


@pytest.mark.parametrize("use_rope,HW,scale1d", [(True, (8, 8), None), (False, (8, 8), None), (True, (12, 8), 2)])
def test_osp_v110_mirror_vs_reference_model(monkeypatch, use_rope, HW, scale1d):
    """videosys_b200's Open-Sora-Plan v1.1.0 front end, its kernel entries replaced by torch stand-ins
    (tests/kernels_emul.py), against the reference's own LatteT2V executed unmodified (oracle/ref_loader.load_osp_v110):
    RoPE tables (2-D / 1-D, linear scaling), position tables, text padding mask, block order, output head."""
    from tests import kernels_emul

    cfg = dict(OSP_SMALL, use_rope=use_rope, interpolation_scale_1d=scale1d)
    B, Fr = 2, 5
    x, enc, m = _osp_inputs(B, Fr, HW)
    t = torch.tensor([500, 500])

    def reference():
        ref = _osp_ref(cfg)
        with torch.no_grad():
            return _template(ref.state_dict()), ref(x, timestep=t, all_timesteps=torch.tensor([900, 500]), encoder_hidden_states=enc,
                                                    added_cond_kwargs={"resolution": None, "aspect_ratio": None},
                                                    attention_mask=torch.ones(B, Fr, *HW), encoder_attention_mask=m,
                                                    return_dict=False)[0]

    tmpl, want = _ref(f"osp_mirror.{use_rope}.{HW[0]}x{HW[1]}.{scale1d}", reference)
    kernels_emul.emulate(monkeypatch)
    net = _osp_net(cfg, tmpl)
    got = net(x, timestep=t, all_timesteps=[900, 500], encoder_hidden_states=enc, attention_mask=torch.ones(B, Fr, *HW),
              encoder_attention_mask=m, return_dict=False)[0]
    got, want = _pair(got, want)
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (got - want).abs().max()


def test_osp_v110_pab_vs_reference_model(monkeypatch):
    """Eight steps with PAB (attention broadcast on all three gates + the MLP skip windows) on both sides."""
    from tests import kernels_emul
    from videosys_b200.core.pab import pab_mgr as ours

    ts = [900, 700, 650, 600, 550, 500, 450, 50]
    mlp = {700: {"block": [0, 1], "skip_count": 2}, 550: {"block": [1], "skip_count": 1}}
    kw = dict(spatial_broadcast=True, spatial_threshold=[100, 850], spatial_range=2, temporal_broadcast=True,
              temporal_threshold=[100, 850], temporal_range=3, cross_broadcast=True, cross_threshold=[100, 850], cross_range=4,
              mlp_broadcast=True, mlp_spatial_broadcast_config=mlp, mlp_temporal_broadcast_config=mlp)
    B, Fr, HW = 2, 5, (8, 8)
    inputs = [_osp_inputs(B, Fr, HW, tag=f"ospp{step}.") for step in range(len(ts))]

    def reference():
        P = ref_loader.load().pab_mgr
        ref = _osp_ref(OSP_SMALL, "ospp.")
        P.set_pab_manager(P.PABConfig(**kw))
        P.update_steps(len(ts))
        outs = []
        try:
            with torch.no_grad():
                for (x, enc, m), t in zip(inputs, ts):
                    outs.append(ref(x, timestep=torch.tensor([t, t]), all_timesteps=torch.tensor(ts), encoder_hidden_states=enc,
                                    added_cond_kwargs={"resolution": None, "aspect_ratio": None},
                                    attention_mask=torch.ones(B, Fr, *HW), encoder_attention_mask=m, return_dict=False)[0])
        finally:
            P.PAB_MANAGER = None
        return _template(ref.state_dict()), outs

    tmpl, refs = _ref("osp_pab.steps", reference)
    kernels_emul.emulate(monkeypatch)
    net = _osp_net(OSP_SMALL, tmpl, "ospp.")
    ours.set_pab_manager(ours.PABConfig(**kw))
    ours.update_steps(len(ts))
    net.reset_pab_state()
    try:
        for step, ((x, enc, m), t) in enumerate(zip(inputs, ts)):
            got = net(x, timestep=torch.tensor([t, t]), all_timesteps=ts, encoder_hidden_states=enc, encoder_attention_mask=m,
                      return_dict=False)[0]
            got, want = _pair(got, refs[step])
            assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (step, (got - want).abs().max())
    finally:
        ours.set_pab_manager(None)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_osp_v110_rope_tables_vs_reference_classes(dtype):
    """The cos / signed-sin tables of vsb_qk_rope_halves against LinearScalingRoPE2D / LinearScalingRoPE1D run on q itself:
    q*cos + partner*sin_signed, evaluated op by op in the dtype, equals the reference's output bit for bit."""
    from videosys_b200.models.transformers.open_sora_plan_v110_transformer_3d import rope_tables

    D, Hh, h, w, Fr = 72, 3, 5, 7, 9
    q2 = synth.normalish("rope.q2", (2, Hh, h * w, D)).to(dtype)
    q1 = synth.normalish("rope.q1", (4, Hh, Fr, D)).to(dtype)

    def reference():
        M = ref_loader.load_osp_v110()
        want2 = M.LinearScalingRoPE2D(scaling_factor=2)(q2, M.PositionGetter2D()(2, h, w, "cpu"))
        return want2, M.LinearScalingRoPE1D(scaling_factor=2)(q1, M.PositionGetter1D()(4, Fr, "cpu"))

    want2, want1 = _ref(f"osp_rope.{dtype}", reference)
    yx = torch.cartesian_prod(torch.arange(h), torch.arange(w))
    c, s, half = rope_tables(D, [yx[:, 0], yx[:, 1]], 2, dtype, "cpu")
    assert half == 18

    def apply(q, c, s, half):
        partner = q.reshape(*q.shape[:-1], D // (2 * half), 2, half).flip(-2).reshape(q.shape)
        return q * c.to(dtype) + partner * s.to(dtype)

    assert torch.equal(*_pair(apply(q2, c, s, half), want2))
    c, s, half = rope_tables(D, [torch.arange(Fr)], 2, dtype, "cpu")
    assert half == 36 and torch.equal(*_pair(apply(q1, c, s, half), want1))


# ---- Latte: oracle and product host logic against the UNMODIFIED reference model ---------------------------------------------
LATTE_SMALL = dict(num_attention_heads=2, attention_head_dim=72, in_channels=4, out_channels=8, num_layers=2,
                   cross_attention_dim=144, attention_bias=True, sample_size=8, patch_size=2, activation_fn="gelu-approximate",
                   norm_type="ada_norm_single", norm_elementwise_affine=False, norm_eps=1e-6, caption_channels=32, video_length=6)
LATTE_SMALL_O = dict(heads=2, head_dim=72, layers=2, patch=2, sample_size=8, out_channels=8, video_length=6)


def _latte_weights(tmpl, dtype, tag="lattep."):
    sd = synth.fill_state_dict({k: v.float() for k, v in tmpl.items()}, tag)
    return {k: v.to(dtype) for k, v in sd.items()}


def _latte_ref(dtype=torch.float32, tag="lattep."):
    ref = ref_loader.build_latte(dtype=dtype, **LATTE_SMALL)
    ref.load_state_dict(_latte_weights(ref.state_dict(), dtype, tag))
    return ref


def _latte_call(ref, x, t, enc, all_ts=(900, 500)):
    return ref(x, timestep=t, all_timesteps=torch.tensor(list(all_ts)), encoder_hidden_states=enc,
               added_cond_kwargs={"resolution": None, "aspect_ratio": None}, enable_temporal_attentions=True,
               return_dict=False)[0]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_latte_oracle_vs_reference_model(dtype):
    """oracle/latte_oracle.transformer_forward against the reference's own LatteT2V (models/transformers/
    latte_transformer_3d.py, executed unmodified; its diffusers leaves = the reference's vendored copies, ref_loader.load_latte):
    the whole forward -- PatchEmbed + 2-D sin-cos table, AdaLayerNormSingle, caption projection, both block kinds,
    temp_pos_embed, output head, un-patchify.  fp32: equal up to summation order; bf16: bit for bit."""
    from oracle import latte_oracle as LO

    x = synth.normalish("lattep.x", (2, 4, 6, 8, 8)).to(dtype)
    enc = synth.normalish("lattep.enc", (2, 7, 32)).to(dtype)
    t = torch.tensor([500, 500])

    def reference():
        ref = _latte_ref(dtype)
        with torch.no_grad():
            return _template(ref.state_dict()), _latte_call(ref, x, t, enc)

    tmpl, want = _ref(f"latte_oracle.{dtype}", reference)
    sd = _latte_weights(_from_template(tmpl), dtype)
    with torch.no_grad():
        got = LO.transformer_forward(sd, LATTE_SMALL_O, x, t, enc)
    got, want = _pair(got, want)
    if dtype == torch.float32:
        assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (got - want).abs().max()
    else:
        print(f"[pin] latte oracle bf16 vs reference bf16: bit-equal {(got == want).float().mean().item()*100:.1f} %")
        _assert_same(got, want, dtype)


def test_latte_mirror_vs_reference_model(monkeypatch):
    """videosys_b200's LatteT2V (kernel entries = torch stand-ins) against the reference model, fp32, incl. 8 PAB steps with the
    MLP skip on both sides."""
    from tests import kernels_emul
    from videosys_b200.core.pab import pab_mgr as ours
    from videosys_b200.models.transformers.latte_transformer_3d import LatteT2V

    x = synth.normalish("lattep.x", (2, 4, 6, 8, 8))
    enc = synth.normalish("lattep.enc", (2, 7, 32))
    t = torch.tensor([500, 500])
    ts = [900, 700, 650, 600, 550, 500, 450, 50]
    xs = [synth.normalish(f"lattep.x{step}", (2, 4, 6, 8, 8)) for step in range(len(ts))]
    mlp = {700: {"block": [0, 1], "skip_count": 2}, 550: {"block": [1], "skip_count": 1}}
    kw = dict(spatial_broadcast=True, spatial_threshold=[100, 800], spatial_range=2, temporal_broadcast=True,
              temporal_threshold=[100, 800], temporal_range=3, cross_broadcast=True, cross_threshold=[100, 800], cross_range=6,
              mlp_broadcast=True, mlp_spatial_broadcast_config=mlp, mlp_temporal_broadcast_config=mlp)

    def reference():
        P = ref_loader.load().pab_mgr
        ref = _latte_ref()
        with torch.no_grad():
            plain = _latte_call(ref, x, t, enc)
        P.set_pab_manager(P.PABConfig(**kw))
        P.update_steps(len(ts))
        outs = []
        try:
            with torch.no_grad():
                for xv, tv in zip(xs, ts):
                    outs.append(_latte_call(ref, xv, torch.tensor([tv, tv]), enc, ts))
        finally:
            P.PAB_MANAGER = None
        return _template(ref.state_dict()), plain, outs

    tmpl, want, refs = _ref("latte_mirror.steps", reference)
    kernels_emul.emulate(monkeypatch)
    net = LatteT2V(**LATTE_SMALL)
    net.load_state_dict(_latte_weights(_from_template(tmpl), torch.float32))
    net.eval()
    got, want = _pair(net(x, timestep=t, all_timesteps=[900, 500], encoder_hidden_states=enc, return_dict=False)[0], want)
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (got - want).abs().max()
    ours.set_pab_manager(ours.PABConfig(**kw))
    ours.update_steps(len(ts))
    net.reset_pab_state()
    try:
        for step, (xv, tv) in enumerate(zip(xs, ts)):
            got = net(xv, timestep=torch.tensor([tv, tv]), all_timesteps=ts, encoder_hidden_states=enc, return_dict=False)[0]
            got, want = _pair(got, refs[step])
            assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (step, (got - want).abs().max())
    finally:
        ours.set_pab_manager(None)


# ---- CogVideoX: oracle and product host logic against the UNMODIFIED reference model ------------------------------------------
COGX_SMALL = dict(num_attention_heads=4, attention_head_dim=64, in_channels=4, out_channels=4, time_embed_dim=64, text_embed_dim=48,
                  num_layers=2, sample_width=16, sample_height=12, sample_frames=9, max_text_seq_length=16)
COGX_SMALL_O = dict(heads=4, head_dim=64, layers=2, patch=2, max_text=16, sample_width=16, sample_height=12, sample_frames=9,
                    out_channels=4)


def _cogx_weights(tmpl, dtype, tag="cogxp."):
    sd = synth.fill_state_dict({k: v.float() for k, v in tmpl.items()}, tag)
    for k in sd:  # LayerNorm weights around 1 (fill_state_dict treats them as matrices)
        if k.endswith("norm.weight") or k.endswith("norm_final.weight") or k.endswith("norm_q.weight") or k.endswith("norm_k.weight"):
            sd[k] = 1.0 + 0.2 * synth.uniform(tag + k, tuple(sd[k].shape))
    return {k: v.to(dtype) for k, v in sd.items()}


def _cogx_ref(dtype=torch.float32, tag="cogxp.", **extra):
    ref = ref_loader.build_cogvideox(dtype=dtype, **dict(COGX_SMALL, **extra))
    ref.load_state_dict(_cogx_weights(ref.state_dict(), dtype, tag))
    return ref


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_cogvideox_oracle_vs_reference_model(dtype):
    """oracle/cogvideox_oracle.transformer_forward against the reference's own CogVideoXTransformer3DModel (executed
    unmodified; diffusers Attention / FeedForward = the reference's vendored copies, ref_loader.load_cogvideox): patch / text
    embedding, position table, LayerNormZero blocks with the joint-attention processor, norm_final + AdaLayerNorm head,
    un-patchify."""
    from oracle import cogvideox_oracle as CO

    lat = synth.normalish("cogxp.lat", (2, 3, 4, 12, 16)).to(dtype)
    txt = synth.normalish("cogxp.txt", (2, 16, 48)).to(dtype)
    ts = torch.tensor([499, 499])

    def reference():
        ref = _cogx_ref(dtype)
        with torch.no_grad():
            return _template(ref.state_dict()), ref(lat, txt, ts, return_dict=False)[0]

    tmpl, want = _ref(f"cogx_oracle.{dtype}", reference)
    sd = _cogx_weights(_from_template(tmpl), dtype)
    with torch.no_grad():
        got = CO.transformer_forward(sd, COGX_SMALL_O, lat, txt, ts)
    got, want = _pair(got, want)
    if dtype == torch.float32:
        assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (got - want).abs().max()
    else:
        print(f"[pin] cogvideox oracle {dtype} vs reference: bit-equal {(got == want).float().mean().item()*100:.1f} %")
        _assert_same(got, want, dtype)


def test_cogvideox_mirror_vs_reference_model(monkeypatch):
    """videosys_b200's CogVideoXTransformer3DModel (kernel entries = torch stand-ins) against the reference model, fp32, plain
    and over 8 PAB steps."""
    from tests import kernels_emul
    from videosys_b200.core.pab import pab_mgr as ours
    from videosys_b200.models.transformers.cogvideox_transformer_3d import CogVideoXTransformer3DModel

    lat = synth.normalish("cogxp.lat", (2, 3, 4, 12, 16))
    txt = synth.normalish("cogxp.txt", (2, 16, 48))
    ts = torch.tensor([499, 499])
    kw = dict(spatial_broadcast=True, spatial_threshold=[100, 850], spatial_range=2)
    steps = [900, 700, 650, 600, 550, 500, 450, 50]
    lats = [synth.normalish(f"cogxp.lat{step}", (2, 3, 4, 12, 16)) for step in range(len(steps))]

    def reference():
        P = ref_loader.load().pab_mgr
        ref = _cogx_ref()
        with torch.no_grad():
            plain = ref(lat, txt, ts, return_dict=False)[0]
        P.set_pab_manager(P.PABConfig(**kw))
        P.update_steps(len(steps))
        outs = []
        try:
            with torch.no_grad():
                for lv, tv in zip(lats, steps):
                    outs.append(ref(lv, txt, torch.tensor([tv, tv]), return_dict=False)[0])
        finally:
            P.PAB_MANAGER = None
        return _template(ref.state_dict()), plain, outs

    tmpl, want, refs = _ref("cogx_mirror.steps", reference)
    kernels_emul.emulate(monkeypatch)
    net = CogVideoXTransformer3DModel(**COGX_SMALL)
    missing, unexpected = net.load_state_dict(_cogx_weights(_from_template(tmpl), torch.float32), strict=False)
    assert not missing and all(".attn1.to_" in k and ("_temp" in k or "_cross" in k or "_context" in k or "temporal" in k)
                               for k in unexpected), (missing, unexpected)  # the vendored Attention's Vchitect-only members
    net.eval()
    got, want = _pair(net(lat, txt, ts, return_dict=False)[0], want)
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (got - want).abs().max()
    ours.set_pab_manager(ours.PABConfig(**kw))
    ours.update_steps(len(steps))
    net.reset_pab_state()
    try:
        for step, (lv, tv) in enumerate(zip(lats, steps)):
            got, want = _pair(net(lv, txt, torch.tensor([tv, tv]), return_dict=False)[0], refs[step])
            assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (step, (got - want).abs().max())
    finally:
        ours.set_pab_manager(None)


# ---- Vchitect: oracle and product host logic against the UNMODIFIED reference transformer ---------------------------------------
VCH_SMALL = dict(sample_size=8, patch_size=2, in_channels=4, num_layers=3, attention_head_dim=64, num_attention_heads=2,
                 joint_attention_dim=48, caption_projection_dim=128, pooled_projection_dim=40, out_channels=4, pos_embed_max_size=12)
VCH_SMALL_O = dict(heads=2, head_dim=64, layers=3, patch=2, sample_size=8, pos_embed_max_size=12, out_channels=4)


def _vch_weights(tmpl, dtype, tag="vchm."):
    sd0 = {k: v.float() for k, v in tmpl.items()}
    sd = synth.fill_state_dict(sd0, tag)
    sd["pos_embed.pos_embed"] = sd0["pos_embed.pos_embed"]  # the sin-cos table is not a weight
    return {k: v.to(dtype) for k, v in sd.items()}


def _vch_ref(dtype=torch.float32, tag="vchm."):
    ref = ref_loader.build_vchitect(dtype=dtype, **VCH_SMALL)
    ref.load_state_dict(_vch_weights(ref.state_dict(), dtype, tag))
    return ref


def _vch_template(ref):
    return _template(ref.state_dict(), keep=("pos_embed.pos_embed",))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("Fr", [5, 1])
def test_vchitect_oracle_vs_reference_model(Fr, dtype):
    """oracle/vchitect_oracle.transformer_forward against the reference's VchitectXLTransformerModel (vchitect_transformer_3d.py
    executed unmodified on the reference's VchitectAttention; five diffusers leaf classes restated in oracle/ref_loader.py):
    per-frame text broadcast in the first block, context_pre_only last block, the three attentions, norm_out, un-patchify."""
    from oracle import vchitect_oracle as VO

    lat = synth.normalish("vchm.lat", (1, Fr, 4, 12, 16)).to(dtype)
    enc = synth.normalish("vchm.enc", (1, 9, 48)).to(dtype)
    pooled = synth.normalish("vchm.pool", (1, 40)).to(dtype)
    ts = torch.tensor([500.0])

    def reference():
        ref = _vch_ref(dtype)
        with torch.no_grad():
            return _vch_template(ref), ref(lat, encoder_hidden_states=enc, pooled_projections=pooled, timestep=ts, return_dict=False)[0]

    tmpl, want = _ref(f"vch_oracle.{Fr}.{dtype}", reference)
    sd = _vch_weights(_from_template(tmpl), dtype)
    with torch.no_grad():
        got = VO.transformer_forward(sd, VCH_SMALL_O, lat, enc, pooled, ts)
    got, want = _pair(got, want)
    if dtype == torch.float32:
        assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (got - want).abs().max()
    else:
        print(f"[pin] vchitect oracle bf16 vs reference: bit-equal {(got == want).float().mean().item()*100:.1f} %")
        _assert_same(got, want, dtype)


def test_vchitect_mirror_vs_reference_model(monkeypatch):
    """videosys_b200's VchitectXLTransformerModel (kernel entries = torch stand-ins) against the reference model: strict
    state-dict compatibility, fp32 forward, and 8 steps with the three PAB gates on both sides."""
    from tests import kernels_emul
    from videosys_b200.core.pab import pab_mgr as ours
    from videosys_b200.models.transformers.vchitect_transformer_3d import VchitectXLTransformerModel

    enc = synth.normalish("vchm.enc", (1, 9, 48))
    pooled = synth.normalish("vchm.pool", (1, 40))
    kw = dict(spatial_broadcast=True, spatial_threshold=[100, 800], spatial_range=2, temporal_broadcast=True,
              temporal_threshold=[100, 800], temporal_range=3, cross_broadcast=True, cross_threshold=[100, 800], cross_range=4)
    runs = {pab: ([900, 700, 650, 600, 550, 500, 450, 50] if pab else [500]) for pab in (False, True)}

    def lat(step):
        return synth.normalish(f"vchm.lat{step}", (1, 4, 4, 12, 16))

    def reference():
        P = ref_loader.load().pab_mgr
        ref = _vch_ref()
        res = {}
        for pab, steps in runs.items():
            if pab:
                P.set_pab_manager(P.PABConfig(**kw))
                P.update_steps(len(steps))
            try:
                with torch.no_grad():
                    res[pab] = [ref(lat(step), encoder_hidden_states=enc, pooled_projections=pooled, timestep=torch.tensor([float(tv)]),
                                    return_dict=False)[0] for step, tv in enumerate(steps)]
            finally:
                P.PAB_MANAGER = None
        return _vch_template(ref), res[False], res[True]

    tmpl, plain, with_pab = _ref("vch_mirror.steps", reference)
    kernels_emul.emulate(monkeypatch)
    net = VchitectXLTransformerModel(**VCH_SMALL)
    net.load_state_dict(_vch_weights(_from_template(tmpl), torch.float32))  # strict
    net.eval()
    for pab, refs in ((False, plain), (True, with_pab)):
        steps = runs[pab]
        if pab:
            ours.set_pab_manager(ours.PABConfig(**kw))
            ours.update_steps(len(steps))
            net.reset_pab_state()
        try:
            for step, tv in enumerate(steps):
                got, want = _pair(net(lat(step), enc, pooled, torch.tensor([float(tv)]), return_dict=False)[0], refs[step])
                assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (pab, step, (got - want).abs().max())
        finally:
            ours.set_pab_manager(None)


def _vch_sp_worker(rank, world, port, Fr, gold, q):
    """gold None: run the reference as well (its checkout is present); else (template, per-rank reference outputs)."""
    import os
    import traceback
    import types

    os.environ["CUDA_VISIBLE_DEVICES"] = ""  # a CPU test: gloo ranks, never NCCL on a shared local GPU
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        import torch.distributed as dist

        from tests import kernels_emul
        from videosys_b200.core.distributed.parallel_mgr import initialize
        from videosys_b200.models.transformers.vchitect_transformer_3d import VchitectXLTransformerModel

        kernels_emul.emulate_global()
        initialize(rank, world)

        def a2a(out_list, in_list, group=None):  # gloo has no all_to_all: the same exchange through all_to_all_single
            send = torch.stack([t.contiguous() for t in in_list])
            recv = torch.empty_like(send)
            dist.all_to_all_single(recv, send, group=group)
            for o, r in zip(out_list, recv.unbind(0)):
                o.copy_(r)

        dist.all_to_all = a2a
        lat = synth.normalish("vchsp.lat", (1, Fr, 4, 12, 16))
        enc = synth.normalish("vchsp.enc", (1, 9, 48))
        pooled = synth.normalish("vchsp.pool", (1, 40))
        ts = torch.tensor([500.0])
        if gold is None:
            RC = ref_loader.load().comm

            def gather_cpu(input_, pg, dim, pad):  # the reference's _gather_sequence_func (comm.py:170-190) minus its CUDA assert
                parts = [torch.empty_like(input_.contiguous()) for _ in range(dist.get_world_size(pg))]
                dist.all_gather(parts, input_.contiguous(), group=pg)
                out = torch.cat(parts, dim=dim)
                return out.narrow(dim, 0, out.size(dim) - pad) if pad > 0 else out

            RC._gather_sequence_func = gather_cpu
            ref = _vch_ref()
            pm = types.SimpleNamespace(sp_size=world, sp_group=dist.group.WORLD, cp_size=1, sp_rank=rank)
            ref.parallel_manager = pm
            for mod in ref.modules():
                if hasattr(mod, "parallel_manager"):
                    mod.parallel_manager = pm
            tmpl = _vch_template(ref)
            with torch.no_grad():
                want = ref(lat, encoder_hidden_states=enc, pooled_projections=pooled, timestep=ts, return_dict=False)[0]
        else:
            tmpl, want = gold[0], gold[1][rank]
        net = VchitectXLTransformerModel(**VCH_SMALL)
        net.load_state_dict(_vch_weights(_from_template(tmpl), torch.float32))
        net.eval()
        net.enable_parallel(1, world, False)
        got = net(lat, enc, pooled, ts, return_dict=False)[0]
        q.put((rank, float((got - want).abs().max()), float(want.abs().max()), tuple(got.shape) == tuple(want.shape), None,
               tmpl, want))
        dist.barrier()
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        q.put((rank, None, None, None, traceback.format_exc(), None, None))


@pytest.mark.parametrize("Fr", [4, 5, 2])  # 5 frames: a zero frame pads the last rank; 2: one frame per rank (temporal branch * 0)
def test_vchitect_sequence_parallel_vs_reference_gloo_world2(Fr):
    """Two gloo ranks, both running videosys_b200's transformer (kernel entries = torch stand-ins) under frame-sharded sequence
    parallelism against the UNMODIFIED reference transformer under the same sharding (run on the ranks where the checkout is
    present, stored per rank otherwise): same output on every rank, incl. the reference's quirks under sp (cross attention
    against the text keys of the rank's own first frame, cur_frame == 1 judged on the local frame count)."""
    import multiprocessing as mp
    import os

    world = 2

    def run(gold):
        port = 30700 + (os.getpid() % 250) + Fr + (0 if gold is None else 5)
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        procs = [ctx.Process(target=_vch_sp_worker, args=(r, world, port, Fr, gold, q)) for r in range(world)]
        [p.start() for p in procs]
        wants, tmpl = [None] * world, None
        for _ in range(world):
            r, err_abs, scale, same_shape, tb, tmpl_r, want = q.get(timeout=300)
            assert tb is None, tb
            assert same_shape and err_abs <= 1e-4 * max(scale, 1.0), (r, err_abs, scale)
            wants[r], tmpl = want, tmpl_r
        [p.join(timeout=60) for p in procs]
        return tmpl, wants

    key = f"vch_sp.{Fr}"
    if ref_loader.available():
        _ref(key, lambda: run(None))
    else:
        run(_ref(key, None))


# ---- Open-Sora-Plan v1.2.0: the product's host logic against the UNMODIFIED reference model --------------------------------
OSP12_SMALL = dict(num_attention_heads=2, attention_head_dim=96, in_channels=4, out_channels=8, num_layers=2, cross_attention_dim=192,
                   attention_bias=True, sample_size=(8, 8), sample_size_t=5, patch_size=2, patch_size_t=1,
                   activation_fn="gelu-approximate", norm_type="ada_norm_single", norm_elementwise_affine=False, norm_eps=1e-6,
                   caption_channels=32, interpolation_scale_h=1.0, interpolation_scale_w=2.0, interpolation_scale_t=1.5,
                   attention_mode="math", downsampler=None, use_rope=True)


def _osp12_ref(cfg, tag="osp12."):
    ref = ref_loader.build_osp_v120(**cfg)
    ref.load_state_dict(synth.fill_state_dict(ref.state_dict(), tag))
    return ref


def _osp12_net(cfg, tmpl, tag="osp12."):
    from videosys_b200.models.transformers.open_sora_plan_v120_transformer_3d import OpenSoraT2V

    net = OpenSoraT2V(**cfg)
    net.load_state_dict(synth.fill_state_dict(_from_template(tmpl), tag))  # strict
    return net.eval()


def _osp12_call(ref, x, t, enc, m):
    return ref(x, timestep=t, encoder_hidden_states=enc, attention_mask=torch.ones(x.shape[0], x.shape[2], x.shape[3], x.shape[4]),
               encoder_attention_mask=m, return_dict=False)[0]


@pytest.mark.parametrize("use_rope,HW", [(True, (8, 8)), (False, (8, 8)), (True, (12, 8))])
def test_osp_v120_mirror_vs_reference_model(monkeypatch, use_rope, HW):
    """videosys_b200's OpenSoraT2V (kernel entries = torch stand-ins) against the reference's own OpenSoraT2V executed
    unmodified: RoPE3D tables with per-axis interpolation scales, absolute position tables when RoPE is off, text padding
    mask, block order, output head / un-patchify."""
    from tests import kernels_emul

    cfg = dict(OSP12_SMALL, use_rope=use_rope)
    x, enc, m = _osp_inputs(2, 5, HW, tag="osp12.")
    t = torch.tensor([500, 500])

    def reference():
        ref = _osp12_ref(cfg)
        with torch.no_grad():
            return _template(ref.state_dict()), _osp12_call(ref, x, t, enc, m)

    tmpl, want = _ref(f"osp12_mirror.{use_rope}.{HW[0]}x{HW[1]}", reference)
    kernels_emul.emulate(monkeypatch)
    net = _osp12_net(cfg, tmpl)
    got = net(x, timestep=t, encoder_hidden_states=enc, encoder_attention_mask=m, return_dict=False)[0]
    got, want = _pair(got, want)
    assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (got - want).abs().max()


def test_osp_v120_pab_vs_reference_model(monkeypatch):
    from tests import kernels_emul
    from videosys_b200.core.pab import pab_mgr as ours

    ts = [900, 700, 650, 600, 550, 500, 450, 50]
    kw = dict(spatial_broadcast=True, spatial_threshold=[100, 850], spatial_range=2, cross_broadcast=True,
              cross_threshold=[100, 850], cross_range=3)
    inputs = [_osp_inputs(2, 5, (8, 8), tag=f"osp12p{step}.") for step in range(len(ts))]

    def reference():
        P = ref_loader.load().pab_mgr
        ref = _osp12_ref(OSP12_SMALL, "osp12p.")
        P.set_pab_manager(P.PABConfig(**kw))
        P.update_steps(len(ts))
        outs = []
        try:
            with torch.no_grad():
                for (x, enc, m), t in zip(inputs, ts):
                    outs.append(_osp12_call(ref, x, torch.tensor([t, t]), enc, m))
        finally:
            P.PAB_MANAGER = None
        return _template(ref.state_dict()), outs

    tmpl, refs = _ref("osp12_pab.steps", reference)
    kernels_emul.emulate(monkeypatch)
    net = _osp12_net(OSP12_SMALL, tmpl, "osp12p.")
    ours.set_pab_manager(ours.PABConfig(**kw))
    ours.update_steps(len(ts))
    net.reset_pab_state()
    try:
        for step, ((x, enc, m), t) in enumerate(zip(inputs, ts)):
            got = net(x, timestep=torch.tensor([t, t]), encoder_hidden_states=enc, encoder_attention_mask=m, return_dict=False)[0]
            got, want = _pair(got, refs[step])
            assert torch.allclose(got, want, rtol=1e-4, atol=1e-5), (step, (got - want).abs().max())
    finally:
        ours.set_pab_manager(None)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_osp_v120_rope3d_tables_vs_reference_class(dtype):
    from videosys_b200.models.transformers.open_sora_plan_v120_transformer_3d import rope3d_tables

    D, Hh, T, h, w = 96, 3, 4, 3, 5
    q = synth.normalish("rope3.q", (2, Hh, T * h * w, D)).to(dtype)

    def reference():
        M = ref_loader.load_osp_v120()
        return M.RoPE3D(interpolation_scale_thw=(1.5, 1.0, 2.0))(q, M.PositionGetter3D()(2, T, h, w, "cpu"))

    want = _ref(f"osp12_rope3d.{dtype}", reference)
    c, s, half = rope3d_tables(D, T, h, w, (1.5, 1.0, 2.0), dtype, "cpu")
    assert half == 16
    partner = q.reshape(*q.shape[:-1], D // (2 * half), 2, half).flip(-2).reshape(q.shape)
    assert torch.equal(*_pair(q * c.to(dtype) + partner * s.to(dtype), want))


def test_stdit3_mirror_vs_reference_model(monkeypatch):
    """The headline model's front end (videosys_b200 STDiT3, kernel entries = torch stand-ins, bf16 as it insists) against
    the reference STDiT3 executed unmodified: within the reference's own bf16-vs-fp32 error, with PAB off and over 6 PAB
    steps (hoisted text projections, modulation tables, per-frame mask select, final layer on the shard, un-patchify)."""
    from tests import kernels_emul
    from videosys_b200.core.pab import pab_mgr as ours
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config

    c = cases.small_model_cfg(depth=2)
    kw = dict(spatial_broadcast=True, spatial_threshold=[100, 930], spatial_range=2, temporal_broadcast=True,
              temporal_threshold=[100, 930], temporal_range=3, cross_broadcast=True, cross_threshold=[100, 930], cross_range=4)
    steps = [900.0, 800.0, 700.0, 600.0, 500.0, 50.0]

    def rel(a, b):
        return ((a.double() - b.double()).norm() / b.double().norm()).item()

    def run(model, inp, dt):
        f = lambda v: v.to(dt) if torch.is_tensor(v) and v.is_floating_point() else v  # noqa: E731
        with torch.no_grad():
            return model(f(inp["x"]), f(inp["timestep"]), f(inp["y"]), mask=inp["mask"], x_mask=inp["x_mask"], fps=f(inp["fps"]),
                         height=f(inp["height"]), width=f(inp["width"]))

    def reference():
        P = ref_loader.load().pab_mgr
        ref16 = ref_loader.build_stdit3(dtype=torch.bfloat16, **c)
        sd = synth.fill_state_dict(ref16.state_dict(), "stde.")
        ref16.load_state_dict(sd)
        ref32 = ref_loader.build_stdit3(dtype=torch.float32, **c)
        ref32.load_state_dict({k: v.float() for k, v in sd.items()})
        inp = cases.forward_inputs(torch.bfloat16)
        res = {"w16": [run(ref16, inp, torch.bfloat16)], "w32": [run(ref32, inp, torch.float32)]}
        try:
            for model, dt, name in ((ref16, torch.bfloat16, "w16"), (ref32, torch.float32, "w32")):
                P.set_pab_manager(P.PABConfig(**kw))
                P.update_steps(len(steps))
                for t in steps:
                    inp["timestep"] = torch.tensor([t, t], dtype=torch.bfloat16)
                    res[name].append(run(model, inp, dt))
                P.PAB_MANAGER = None
        finally:
            P.PAB_MANAGER = None
        return _template(ref16.state_dict()), res["w16"], res["w32"]

    tmpl, r16, r32 = _ref("stdit3_mirror.steps", reference)
    kernels_emul.emulate(monkeypatch)
    net = STDiT3(STDiT3Config(**c)).to(torch.bfloat16)
    net.load_state_dict(synth.fill_state_dict(_from_template(tmpl), "stde."))
    net.eval()
    inp = cases.forward_inputs(torch.bfloat16)
    outs = [run(net, inp, torch.bfloat16)]
    ours.set_pab_manager(ours.PABConfig(**kw))
    ours.update_steps(len(steps))
    net.reset_pab_state()
    try:
        for t in steps:
            inp["timestep"] = torch.tensor([t, t], dtype=torch.bfloat16)
            outs.append(run(net, inp, torch.bfloat16))
    finally:
        ours.set_pab_manager(None)
    for i in range(len(outs)):  # i = 0: PAB off; 1..6: the PAB steps
        got, w32 = _pair(outs[i], r32[i])
        _, w16 = _pair(outs[i], r16[i])
        assert rel(got, w32) <= 1.3 * rel(w16, w32) + 1e-4, (i, rel(got, w32), rel(w16, w32))


# ---- CogVideoX-5b: rotary position embeddings ------------------------------------------------------------------------------------
def _cogx_rotary(T=3, gh=6, gw=8, D=64):
    from oracle import cogvideox_oracle as CO

    return CO.rotary_3d(D, CO.resize_crop_region_for_grid((gh, gw), 45, 30), (gh, gw), T)


def test_cogvideox_rotary_helpers_vs_reference():
    """oracle rotary_3d / resize_crop_region_for_grid / apply_rotary_emb and the pipeline mirror's
    _prepare_rotary_positional_embeddings against the reference's own functions (models/modules/embeddings.py:283-412,
    pipelines/cogvideox/pipeline_cogvideox.py:758-773 -- the pipeline module itself needs diffusers: its crop helper is
    compared through its published formula on the oracle side)."""
    from oracle import cogvideox_oracle as CO
    from videosys_b200.pipelines.cogvideox.pipeline_cogvideox import CogVideoXPipeline

    grids = ((30, 45), (6, 8), (20, 20), (9, 40))
    xs = {dtype: synth.normalish("rot.x", (2, 3, 3 * 6 * 8, 64)).to(dtype) for dtype in (torch.float32, torch.bfloat16)}

    def reference():
        import importlib

        ref_loader.load_cogvideox()
        E = importlib.import_module("videosys.models.modules.embeddings")
        tables = [E.get_3d_rotary_pos_embed(64, CO.resize_crop_region_for_grid(g, 45, 30), g, 5, use_real=True) for g in grids]
        c, s = _cogx_rotary()
        return tables, [E.apply_rotary_emb(xs[dt], (c, s)) for dt in (torch.float32, torch.bfloat16)]

    tables, applied = _ref("cogx_rotary.helpers", reference)
    for (gh, gw), (rc, rs) in zip(grids, tables):
        oc, os_ = CO.rotary_3d(64, CO.resize_crop_region_for_grid((gh, gw), 45, 30), (gh, gw), 5)
        assert torch.equal(*_pair(oc, rc)) and torch.equal(*_pair(os_, rs))
        pipe = CogVideoXPipeline.__new__(CogVideoXPipeline)
        pipe.transformer = type("T", (), {"config": type("C", (), {"patch_size": 2, "attention_head_dim": 64})()})()
        pc, ps = pipe._prepare_rotary_positional_embeddings(gh * 16, gw * 16, 5, "cpu")
        assert torch.equal(*_pair(pc, rc)) and torch.equal(*_pair(ps, rs))
    c, s = _cogx_rotary()
    for dt, want in zip((torch.float32, torch.bfloat16), applied):
        assert torch.equal(*_pair(CO.apply_rotary_emb(xs[dt], c, s), want))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_cogvideox_rotary_oracle_and_mirror_vs_reference_model(monkeypatch, dtype):
    """use_rotary_positional_embeddings=True (CogVideoX-5b): oracle forward (bf16 bit for bit) and, in fp32, the product front end
    on the kernel stand-ins (identity rope rows for the text tokens, RoPE-only pre-pass) against the reference model."""
    from oracle import cogvideox_oracle as CO
    from tests import kernels_emul
    from videosys_b200.models.transformers.cogvideox_transformer_3d import CogVideoXTransformer3DModel

    cfg = dict(COGX_SMALL, use_rotary_positional_embeddings=True)
    lat = synth.normalish("cogxr.lat", (2, 3, 4, 12, 16)).to(dtype)
    txt = synth.normalish("cogxr.txt", (2, 16, 48)).to(dtype)
    ts = torch.tensor([499, 499])
    rot = _cogx_rotary()

    def reference():
        ref = _cogx_ref(dtype, "cogxr.", use_rotary_positional_embeddings=True)
        with torch.no_grad():
            return _template(ref.state_dict()), ref(lat, txt, ts, image_rotary_emb=rot, return_dict=False)[0]

    tmpl, want = _ref(f"cogx_rotary_model.{dtype}", reference)
    sd = _cogx_weights(_from_template(tmpl), dtype, "cogxr.")
    with torch.no_grad():
        got = CO.transformer_forward(sd, COGX_SMALL_O, lat, txt, ts, rotary=rot)
    if dtype == torch.float32:
        g, w = _pair(got, want)
        assert torch.allclose(g, w, rtol=1e-4, atol=1e-5), (g - w).abs().max()
        kernels_emul.emulate(monkeypatch)
        net = CogVideoXTransformer3DModel(**cfg)
        missing, unexpected = net.load_state_dict(sd, strict=False)
        assert not missing
        out, w = _pair(net.eval()(lat, txt, ts, image_rotary_emb=rot, return_dict=False)[0], want)
        assert torch.allclose(out, w, rtol=1e-4, atol=1e-5), (out - w).abs().max()
    else:
        _assert_same(got, want, dtype)
