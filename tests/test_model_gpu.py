"""STDiT3 on the sm_90a kernels (videosys_b200) against the oracle and the reference's golden vectors.

End-to-end tolerance (SURVEY.md fact 11 / BASELINE.md section 4): rtol 1e-3 is below one bf16 ulp, and the
reference in bf16 is itself only within that band of its own fp32 run on a few % of elements.  So:
  * per block: output within a few bf16 ulps of the oracle's bf16 block on identical inputs (and mostly bit-equal);
  * per step : ||ours_bf16 - ref_fp32|| <= 1.25 * ||ref_bf16 - ref_fp32||, i.e. no worse than the reference's own
    bf16 error, with the raw rtol/atol pass-rate printed beside the reference's own pass-rate.
"""
import os

import pytest
import torch

from oracle import cases, pab_oracle, stdit3_oracle as O, synth
from tests.helpers import stdit3_state_dict_template

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _build(cfg, tag="golden."):
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config

    dev = _dev()
    sd = synth.fill_state_dict(stdit3_state_dict_template(cfg, BF), tag)
    net = STDiT3(STDiT3Config(**cfg)).to(BF)
    missing = net.load_state_dict(sd, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    return net.to(dev).eval(), sd


def _to(inp, dev):
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in inp.items()}


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _passrate(a, b):
    return torch.isclose(a.float(), b.float(), rtol=1e-3, atol=1e-5).float().mean().item()


@pytest.mark.parametrize("kind", ["spatial", "temporal"])
def test_block_vs_golden_and_oracle(golden_dir, kind):
    gold = torch.load(os.path.join(golden_dir, "stdit3_small.pt"))
    cfg = cases.small_model_cfg(depth=1)
    net, sd = _build(cfg)
    dev = _dev()
    b = cases.block_inputs(BF)
    B, T, S = 2, b["T"], b["S"]
    blk = getattr(net, kind + "_blocks")[0]
    x = b["x"].to(dev).clone()
    mask_u8 = b["x_mask"].to(torch.uint8).to(dev)
    text = dict(y_tok=b["y"].to(dev).reshape(-1, cfg["hidden_size"]).contiguous(), Lv=b["y"].shape[1] // B, kv_lens=None, kv={})
    out = net._run_block(blk, x, text, b["t"].to(dev), b["t0"].to(dev), mask_u8, B, T, S, T, S).cpu()
    ref = gold[f"block_{kind}_bf16"]
    temporal = kind == "temporal"
    orc = O.stdit3_block(sd, f"{kind}_blocks.0.", b["x"], b["y"], b["t"], b["y_lens"], b["x_mask"], b["t0"], T, S,
                         cfg["num_heads"], temporal, sd["rope.freqs"] if temporal else None)
    eq_ref = (out.float() == ref.float()).float().mean().item()
    d = (out.float() - ref.float()).abs()
    mag = torch.maximum(ref.float().abs(), 0.25 * ref.float().abs().amax(dim=-1, keepdim=True))  # ulp at row scale
    ulp = torch.ldexp(torch.ones_like(d), torch.frexp(mag)[1] - 8)
    print(f"[parity] block {kind}: bit-equal to reference golden {eq_ref*100:.2f} %, max {((d/ulp).max().item()):.1f} ulp, "
          f"rel L2 {_rel(out, ref):.3e}; oracle-vs-golden rel L2 {_rel(orc, ref):.3e}")
    assert eq_ref > 0.60  # flash-attention rounding differs from the CPU SDPA the golden was made with
    assert (d / ulp).max().item() <= 8.0
    assert _rel(out, ref) < 4e-3


def test_forward_vs_reference_golden(golden_dir):
    gold = torch.load(os.path.join(golden_dir, "stdit3_small.pt"))
    cfg = cases.small_model_cfg(depth=1)
    net, sd = _build(cfg)
    dev = _dev()
    inp = cases.forward_inputs(BF)
    out = net(**_to(inp, dev)).cpu()
    ref32, ref16 = gold["forward_fp32"].float(), gold["forward_bf16"].float()
    e_ours, e_ref = _rel(out, ref32), _rel(ref16, ref32)
    print(f"[parity] forward small: ||ours-ref_fp32||/||ref|| = {e_ours:.3e}  vs reference bf16 self-error {e_ref:.3e}; "
          f"rtol1e-3/atol1e-5 pass-rate ours-vs-ref_bf16 {_passrate(out, ref16)*100:.1f} %, "
          f"ref_bf16-vs-ref_fp32 {_passrate(ref16, ref32)*100:.1f} %, ours-vs-ref_fp32 {_passrate(out, ref32)*100:.1f} %")
    assert out.shape == ref32.shape and out.dtype == torch.float32
    assert e_ours <= 1.25 * e_ref + 1e-4


def test_forward_depth2_vs_oracle_fullwidth():
    """hidden 1152 / 16 heads (the real block width), depth 2, 240p-like ragged grid (W padded to even)."""
    cfg = dict(hidden_size=1152, num_heads=16, depth=2, caption_channels=256, model_max_length=40)
    net, sd = _build(cfg, tag="full.")
    dev = _dev()
    inp = cases.forward_inputs(BF, B=2, T=6, H=14, W=11, L=40, n_valid=33, cap=256)
    out = net(**_to(inp, dev)).cpu()
    ocfg = cases.oracle_cfg(cfg)
    with torch.no_grad():
        ref16 = O.stdit3_forward(sd, ocfg, **inp)
        sd32 = {k: v.float() for k, v in sd.items()}
        inp32 = {k: (v.float() if torch.is_tensor(v) and v.dtype == BF else v) for k, v in inp.items()}
        ref32 = O.stdit3_forward(sd32, ocfg, **inp32)
    e_ours, e_ref = _rel(out, ref32), _rel(ref16, ref32)
    print(f"[parity] forward 1152x2: ours-vs-fp32 {e_ours:.3e}, oracle bf16-vs-fp32 {e_ref:.3e}, "
          f"pass-rate ours-vs-oracle_bf16 {_passrate(out, ref16)*100:.1f} %, oracle_bf16-vs-fp32 {_passrate(ref16, ref32)*100:.1f} %")
    assert e_ours <= 1.25 * e_ref + 1e-4


def test_pab_schedule_and_replay_over_steps():
    """PAB on: the skip decisions are bit-exact (integer gate) and replayed tensors are the cached ones."""
    from videosys_b200.core.pab import pab_mgr as P

    cfg = cases.small_model_cfg(depth=2)
    net, sd = _build(cfg)
    dev = _dev()
    steps = [1000, 900, 860, 800, 700, 600, 500, 300]
    P.set_pab_manager(P.PABConfig(spatial_broadcast=True, spatial_threshold=[450, 930], spatial_range=2,
                                  temporal_broadcast=True, temporal_threshold=[450, 930], temporal_range=4,
                                  cross_broadcast=True, cross_threshold=[450, 930], cross_range=6))
    P.update_steps(len(steps))
    gate = pab_oracle.opensora_default(len(steps))
    states = {k: [O.BlockPABState() for _ in range(2)] for k in ("spatial", "temporal")}
    states32 = {k: [O.BlockPABState() for _ in range(2)] for k in ("spatial", "temporal")}
    inp = cases.forward_inputs(BF)
    try:
        for i, t in enumerate(steps):
            inp["x"] = synth.normalish(f"pab.x{i}", tuple(inp["x"].shape))
            inp["timestep"] = torch.tensor([float(t)] * 2)
            before = {k: [(b.attn_count, b.cross_count) for b in getattr(net, k + "_blocks")] for k in states}
            launches0 = _launches()
            out = net(**_to(inp, dev)).cpu()
            n_launch = _launches() - launches0
            with torch.no_grad():
                ref = O.stdit3_forward(sd, cases.oracle_cfg(cfg), pab=gate, pab_states=states, **inp)
            for k in states:
                for b, s in zip(getattr(net, k + "_blocks"), states[k]):
                    assert (b.attn_count, b.cross_count) == (s.attn_count, s.cross_count), f"step {i} counters"
            with torch.no_grad():  # the oracle's own bf16 error on this step: bf16 forward vs fp32 forward, same PAB history
                ref32 = O.stdit3_forward({k: v.float() for k, v in sd.items()}, cases.oracle_cfg(cfg), pab=gate,
                                         pab_states=states32, **{k: (v.float() if torch.is_tensor(v) and v.dtype == BF else v)
                                                                 for k, v in inp.items()})
            e_ours, e_ref = _rel(out, ref32), _rel(ref, ref32)
            print(f"[parity] PAB step {i} t={t}: ours-vs-fp32 {e_ours:.3e}, oracle bf16-vs-fp32 {e_ref:.3e}, "
                  f"rel L2 vs oracle bf16 {_rel(out, ref):.3e}, kernels launched {n_launch}")
            assert e_ours <= 1.25 * e_ref + 1e-4
            del before
    finally:
        P.set_pab_manager(None)
        net.reset_pab_state()


def _launches():
    from videosys_b200 import kernels

    return kernels.launch_count()


def test_cpu_tensors_are_rejected():
    """The product path has no CPU fallback: it must fail loudly."""
    from videosys_b200 import kernels
    from videosys_b200._lib import VsbError

    _dev()
    with pytest.raises(VsbError):
        kernels.residual_add(torch.zeros(8, dtype=BF), torch.zeros(8, dtype=BF))


# ---- real shapes (VERDICT r1 "What's weak" 1b): the BASELINE configs' own sequence lengths and width -------------------
def _block_case(tag, B, T, S, L, C=1152, H=16):
    """One (spatial, temporal) block pair at hidden 1152 / 16 heads x 72 with deterministic weights."""
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config

    dev = _dev()
    cfg = dict(hidden_size=C, num_heads=H, depth=1, caption_channels=64, model_max_length=L)
    sd = synth.fill_state_dict(stdit3_state_dict_template(cfg, BF), tag)
    net = STDiT3(STDiT3Config(**cfg)).to(BF)
    net.load_state_dict(sd)
    net = net.to(dev).eval()
    b = cases.block_inputs(BF, C=C, B=B, T=T, S=S, L=L, tag=tag)
    return net, sd, b, dev


def _run_pair(net, sd, b, dev, kinds, B, T, S, C=1152, H=16):
    """Runs the blocks on the GPU; returns (ours, oracle in bf16, oracle in fp32) after the last block."""
    x = b["x"].to(dev).clone()
    mask_u8 = b["x_mask"].to(torch.uint8).to(dev)
    text = dict(y_tok=b["y"].to(dev).reshape(-1, C).contiguous(), Lv=b["y"].shape[1] // B, kv_lens=None, kv={})
    want, want32 = b["x"], b["x"].float()
    sd32 = {k: v.float() for k, v in sd.items()}
    for kind in kinds:
        blk = getattr(net, kind + "_blocks")[0]
        x = net._run_block(blk, x, text, b["t"].to(dev), b["t0"].to(dev), mask_u8, B, T, S, T, S)
        temporal = kind == "temporal"
        with torch.no_grad():
            want = O.stdit3_block(sd, f"{kind}_blocks.0.", want, b["y"], b["t"], b["y_lens"], b["x_mask"], b["t0"], T, S, H,
                                  temporal, sd["rope.freqs"] if temporal else None)
            want32 = O.stdit3_block(sd32, f"{kind}_blocks.0.", want32, b["y"].float(), b["t"].float(), b["y_lens"], b["x_mask"],
                                    b["t0"].float(), T, S, H, temporal, sd32["rope.freqs"] if temporal else None)
    return x.cpu(), want, want32


def _block_report(name, got, want, want32, strict=False):
    """Small shapes (strict): mostly bit-equal to the bf16 oracle, a few ulps at most.  Real shapes: thousands of terms
    per reduction, so the bf16 oracle itself sits ~1e-2 from its fp32 run and two correct bf16 evaluations agree on few
    bits; the gate is the end-to-end criterion: no further from the fp32 oracle than the bf16 oracle is (x 1.25)."""
    eq = (got.float() == want.float()).float().mean().item()
    d = (got.float() - want.float()).abs()
    mag = torch.maximum(want.float().abs(), 0.25 * want.float().abs().amax(dim=-1, keepdim=True))
    ulp = torch.ldexp(torch.ones_like(d), torch.frexp(mag)[1] - 8)
    e_ours, e_ref = _rel(got, want32), _rel(want, want32)
    print(f"[parity] {name}: ours-vs-fp32 oracle {e_ours:.3e}, bf16 oracle-vs-fp32 oracle {e_ref:.3e}; bit-equal to the bf16 "
          f"oracle {eq*100:.2f} %, max {(d/ulp).max().item():.1f} ulp, rel L2 vs bf16 oracle {_rel(got, want):.3e}")
    assert e_ours <= 1.25 * e_ref + 1e-4
    if strict:
        assert eq > 0.60 and (d / ulp).max().item() <= 8.0 and _rel(got, want) < 4e-3


def test_block_pair_240p_real_shape():
    """cfg2's own shapes: CFG batch 2, T = 15 latent frames, S = 15 x 27 = 405 patches, 300 text tokens, hidden 1152:
    one spatial + one temporal block against oracle.stdit3_block (about a second of CPU oracle)."""
    B, T, S, L = 2, 15, 405, 300
    net, sd, b, dev = _block_case("r240.", B, T, S, L)
    got, want, want32 = _run_pair(net, sd, b, dev, ("spatial", "temporal"), B, T, S)
    _block_report("240p block pair [2,15,405,1152]", got, want, want32)


def test_spatial_block_720p_sequence():
    """cfg3's spatial sequence: S = 45 x 80 = 3600 patches (57 key tiles, ragged last query pair) on 2 of the 20 latent
    frames, CFG batch 2, 300 text tokens: one spatial block against oracle.stdit3_block."""
    B, T, S, L = 2, 2, 3600, 300
    net, sd, b, dev = _block_case("r720.", B, T, S, L)
    got, want, want32 = _run_pair(net, sd, b, dev, ("spatial",), B, T, S)
    _block_report("720p spatial block [2,2,3600,1152]", got, want, want32)


@pytest.mark.parametrize("T", [30, 34])
def test_temporal_block_long_video(T):
    """102-frame ("4s") videos give 30 latent frames: temporal attention leaves native_attention for SDPA in the reference
    (attentions.py:95-100); here the RoPE/RMSNorm pre-pass + the flash kernel over strided views."""
    B, S, L = 2, 24, 20
    net, sd, b, dev = _block_case(f"long{T}.", B, T, S, L, C=288, H=4)
    got, want, want32 = _run_pair(net, sd, b, dev, ("temporal",), B, T, S, C=288, H=4)
    _block_report(f"temporal block T={T}", got, want, want32, strict=True)


@pytest.mark.parametrize("flash", [False, True])
def test_cross_attention_unequal_caption_lengths(flash):
    """Two samples with different caption lengths (mask rows of 9 and 15 tokens of 20).
    enable_flash_attn=False: the reference's torch_impl VIEWS the packed tokens as [B, sum/B] (attentions.py:259-262),
    so the slices cross sample boundaries -- reproduced bit-for-bit in addressing; enable_flash_attn=True: varlen
    attention over each sample's own tokens (attentions.py:240-257)."""
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config

    dev = _dev()
    cfg = cases.small_model_cfg(depth=1)
    sd = synth.fill_state_dict(stdit3_state_dict_template(cfg, BF), "golden.")
    net = STDiT3(STDiT3Config(enable_flash_attn=flash, **cfg)).to(BF)
    net.load_state_dict(sd)
    net = net.to(dev).eval()
    inp = cases.forward_inputs(BF)
    mask = torch.zeros(2, 20, dtype=torch.long)
    mask[0, :9] = 1
    mask[1, :15] = 1
    inp["mask"] = mask
    out = net(**_to(inp, dev)).cpu()
    ocfg = cases.oracle_cfg(cfg)
    with torch.no_grad():
        ref16 = O.stdit3_forward(sd, ocfg, cross_varlen=flash, **inp)
        other = O.stdit3_forward(sd, ocfg, cross_varlen=not flash, **inp)
        inp32 = {k: (v.float() if torch.is_tensor(v) and v.dtype == BF else v) for k, v in inp.items()}
        ref32 = O.stdit3_forward({k: v.float() for k, v in sd.items()}, ocfg, cross_varlen=flash, **inp32)
    e_ours, e_ref, e_other = _rel(out, ref32), _rel(ref16, ref32), _rel(other, ref32)
    print(f"[parity] unequal captions flash={flash}: ours-vs-fp32 {e_ours:.3e}, oracle bf16-vs-fp32 {e_ref:.3e}, "
          f"the OTHER addressing vs this fp32 {e_other:.3e}")
    assert e_other > 2 * e_ref, "the two key addressings must differ on this input for the test to mean anything"
    assert e_ours <= 1.25 * e_ref + 1e-4


def test_step_graph_replay_is_bit_identical():
    """core/graph_step.py: eager, captured and replayed denoising steps give the same latents bit for bit, without and
    with PAB (one graph per skip pattern; the counters advance on the host, the caches persist across graphs)."""
    from videosys_b200.core.graph_step import StepGraph
    from videosys_b200.core.pab import pab_mgr as P

    cfg = cases.small_model_cfg(depth=2)
    net, sd = _build(cfg)
    dev = _dev()
    inp = _to(cases.forward_inputs(BF), dev)
    fwd = {k: v for k, v in inp.items() if k not in ("x", "timestep")}
    z0 = inp["x"][:1].to(BF).contiguous()
    ts = [torch.tensor([float(v)], device=dev) for v in (1000, 900, 860, 800, 700, 600, 500, 300, 200, 100)]
    dts = [torch.tensor([0.05], device=dev) for _ in ts]

    def run(graph, pab):
        P.set_pab_manager(P.PABConfig(spatial_broadcast=True, spatial_threshold=[450, 930], spatial_range=2,
                                      temporal_broadcast=True, temporal_threshold=[450, 930], temporal_range=4,
                                      cross_broadcast=True, cross_threshold=[450, 930], cross_range=6) if pab else None)
        P.update_steps(len(ts))
        net.reset_pab_state()
        st = StepGraph(net, 7.0, enabled=graph)
        z, outs = z0.clone(), []
        for rep_ in range(2):  # second pass over the schedule: every pattern now replays its graph
            net.reset_pab_state()
            z = z0.clone()
            for i, t in enumerate(ts):
                z = st.step(z, t, dts[i], fwd, ts_int=int(t.item()))
                outs.append(z.clone())
        return outs, st

    try:
        for pab in (False, True):
            eager, _ = run(False, pab)
            graphed, st = run(True, pab)
            assert st.replays >= len(ts), "the graph path was not taken"
            n = len(ts)
            if not pab:  # without PAB history the second pass over the schedule must reproduce the first, in each mode
                for i in range(n):
                    assert torch.equal(eager[i], eager[i + n]), f"EAGER is not deterministic: step {i} differs between passes"
                    assert torch.equal(graphed[i], graphed[i + n]), f"GRAPH replay is not deterministic: step {i}"
            for i, (a, b) in enumerate(zip(eager, graphed)):
                assert torch.equal(a, b), (f"pab={pab} step {i}: replayed graph differs from eager: max abs diff "
                                           f"{(a.float() - b.float()).abs().max().item():.3e}, "
                                           f"{(a != b).float().mean().item() * 100:.2f} % of the elements")
            print(f"[parity] step graph pab={pab}: {len(st._graphs)} graphs, {st.replays} replays, bit-identical to eager")
    finally:
        P.set_pab_manager(None)
        net.reset_pab_state()


def test_forward_is_deterministic():
    """The same forward, 25 times: bit-identical outputs (no kernel may depend on scheduling order or timing)."""
    cfg = cases.small_model_cfg(depth=2)
    net, sd = _build(cfg)
    dev = _dev()
    inp = _to(cases.forward_inputs(BF), dev)
    ref = net(**inp)
    bad = [i for i in range(25) if not torch.equal(net(**inp), ref)]
    assert not bad, f"forward differs from its first run on repetitions {bad}"
