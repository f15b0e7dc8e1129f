"""FP8 Linears without a GPU: the quantization rule against an explicit round-to-nearest-even e4m3 encoder, and the
STDiT3 front end in FP8 mode on the kernel stand-ins (tests/kernels_emul_fp8.py) against the oracle whose block Linears
STDiT3.FP8_LINEARS (qkv and fc1) are the same fake-quant Linear (tests/fp8_rule.py)."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cases, stdit3_oracle as O, synth
from tests import fp8_rule, kernels_emul_fp8

BF = torch.bfloat16
FP8 = ("attn.qkv", "mlp.fc1")  # STDiT3.FP8_LINEARS


# ---- the rule ----------------------------------------------------------------------------------------------------------
def _e4m3_rne(v):
    """Nearest e4m3 value of float64 v (|v| <= 464), ties to even: 3 fraction bits, exponents -6..8, subnormal step 2^-9."""
    a = np.abs(v)
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    e = np.maximum(e, -6.0)
    q = np.exp2(e - 3)
    return np.copysign(np.round(a / q) * q, v)  # np.round: half to even; the sign of zero kept


def _rows(dtype):
    g = torch.Generator().manual_seed(7)
    x = torch.randn(40, 264, generator=g)
    x[8:16] *= torch.exp2(torch.randint(-24, 12, (264,), generator=g).float())  # wide dynamic range (finite in fp16)
    x[16:20] = 0  # all-zero rows
    x[20:28] *= 1e-4
    x[20:28, 5] = -2000.0  # one outlier
    x[28:32] = torch.exp2(torch.randint(-12, 12, (4, 264), generator=g).float()) * 1.0625  # ties of the e4m3 rounding
    return x.to(dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_quant_rule_codes_and_scales(dtype):
    x = _rows(dtype)
    q, s = fp8_rule.quant_rows(x)
    xf = x.double().numpy()
    amax = np.abs(xf).max(1, keepdims=True)
    nz = amax > 0
    s32 = np.where(nz, np.float32(448.0) / np.where(nz, amax, 1).astype(np.float32), 0).astype(np.float32)  # fp32 448 / amax
    prod = (x.float().numpy() * s32).astype(np.float64)  # the fp32 product the kernel converts
    assert np.abs(prod).max() <= 448.0 * (1 + 2.0**-23)
    want = np.where(nz, _e4m3_rne(prod), 0.0)
    got = q.float().double().numpy()
    assert np.array_equal(got, want)
    assert np.array_equal(np.signbit(got[nz[:, 0]]), np.signbit(want[nz[:, 0]]))
    assert bool((q.view(torch.uint8)[16:20] == 0).all())
    want_s = np.where(nz[:, 0], (amax[:, 0].astype(np.float32) / np.float32(448.0)), 1.0).astype(np.float32)
    assert np.array_equal(s.numpy(), want_s)
    assert not torch.isnan(q.float()).any()


# ---- the front end -----------------------------------------------------------------------------------------------------
def _net(tag="fp8.", depth=2):
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config

    net = STDiT3(STDiT3Config(**cases.small_model_cfg(depth=depth))).to(BF)
    net.load_state_dict(synth.fill_state_dict(net.state_dict(), tag))
    return net.eval()


def _run(net, inp, **kw):
    with torch.no_grad():
        return net(inp["x"].to(BF), inp["timestep"].to(BF), inp["y"].to(BF), mask=inp["mask"], x_mask=inp["x_mask"],
                   fps=inp["fps"], height=inp["height"], width=inp["width"], **kw)


def _oracle(sd, cfg, inp, fp8, monkeypatch):
    six = {id(sd[f"{b}_blocks.{i}.{n}.weight"]) for b in ("spatial", "temporal") for i in range(cfg["depth"]) for n in FP8}

    def linear(x, w, b=None):
        if fp8 and id(w) in six:
            return fp8_rule.fake_quant_linear(x, w, b).to(x.dtype)
        return _linear32(x, w, b)

    ns = {k: getattr(F, k) for k in dir(F) if not k.startswith("_")}
    ns["linear"] = linear
    monkeypatch.setattr(O, "F", types.SimpleNamespace(**ns))
    with torch.no_grad():
        return O.stdit3_forward(sd, cases.oracle_cfg(cfg), **inp)


def _linear32(x, w, b=None):
    """A Linear as the kernels compute it: fp32 products and sum, + bias, one rounding to the 16-bit dtype."""
    y = x.float() @ w.float().T
    return (y if b is None else y + b.float()).to(x.dtype)


def _gemm32(monkeypatch):
    """The bf16 GEMM stand-ins with _linear32 in place of the 16-bit torch Linear."""
    from tests import kernels_emul
    from videosys_b200 import kernels

    monkeypatch.setattr(kernels_emul, "F", types.SimpleNamespace(**{**{k: getattr(F, k) for k in dir(F) if not k.startswith("_")},
                                                                    "linear": _linear32}))
    monkeypatch.setattr(kernels, "gemm_bias_act", kernels_emul.gemm_bias_act)


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def test_fp8_front_end_matches_fake_quant_oracle(monkeypatch):
    """With every Linear evaluated as the kernels do (fp32 sums, one rounding), FP8 mode == the oracle with exactly qkv
    and fc1 of every block fake-quantized, bit for bit, as the bf16 mode == the plain oracle; the two modes differ."""
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3

    assert tuple(".".join(p) for p in STDiT3.FP8_LINEARS) == FP8
    kernels_emul_fp8.emulate(monkeypatch)
    _gemm32(monkeypatch)
    cfg = cases.small_model_cfg(depth=2)
    net = _net()
    sd = net.state_dict()
    inp = cases.forward_inputs(BF)
    bf_out = _run(net, inp)
    net.set_fp8_linears(True)
    fp_out = _run(net, inp)
    ref_bf = _oracle(sd, cfg, inp, False, monkeypatch)
    ref_fp = _oracle(sd, cfg, inp, True, monkeypatch)
    d_bf, d_fp, d_cross = _rel(bf_out, ref_bf), _rel(fp_out, ref_fp), _rel(fp_out, ref_bf)
    print(f"bf16 mode vs bf16 oracle {d_bf:.3e}; fp8 mode vs fake-quant oracle {d_fp:.3e}; fp8 mode vs bf16 oracle {d_cross:.3e}")
    assert torch.equal(bf_out, ref_bf) and torch.equal(fp_out, ref_fp)
    assert d_cross > 1e-3
    names = {n for n, b in net.named_buffers() if n.endswith("fp8_weight")}
    want = {f"{b}_blocks.{i}.{n}.fp8_weight" for b in ("spatial", "temporal") for i in range(2) for n in FP8}
    assert names == want  # kv_linear, the embedders, t_block and the final layer have no e4m3 copy


def test_fp8_state_dict_cache_and_toggle(monkeypatch):
    kernels_emul_fp8.emulate(monkeypatch)
    net = _net()
    inp = cases.forward_inputs(BF)
    sd0 = {k: v.clone() for k, v in net.state_dict().items()}
    bf_out = _run(net, inp)
    net.set_fp8_linears(True)
    fp_out = _run(net, inp)
    sd1 = net.state_dict()
    assert list(sd1) == list(sd0) and all(torch.equal(sd1[k], sd0[k]) for k in sd0)  # keys, shapes, values
    # new weights: the quantized copies follow at the next forward
    net.load_state_dict(synth.fill_state_dict(net.state_dict(), "fp8.other."))
    _run(net, inp)
    for lin in net._fp8_modules():
        q, s = fp8_rule.quant_rows(lin.weight)
        assert torch.equal(lin.fp8_weight, q.view(torch.uint8)) and torch.equal(lin.fp8_scale, s)
    net.load_state_dict(sd0)
    assert torch.equal(_run(net, inp), fp_out)
    # off: the bf16 calls again, bit for bit those of a model on which FP8 was never enabled
    net.set_fp8_linears(False)
    assert torch.equal(_run(net, inp), bf_out)
    assert not any(n.endswith(("fp8_weight", "fp8_scale")) for n, _ in net.named_buffers())
    # a dtype conversion of the module turns the scale buffer to bf16: re-quantized, not served stale
    net.set_fp8_linears(True)
    _run(net, inp)
    net.to(BF)
    lin = net.spatial_blocks[0].attn.qkv
    assert torch.equal(_run(net, inp), fp_out)
    assert lin.fp8_scale.dtype == torch.float32


def test_fp8_pab_plans_unchanged(monkeypatch):
    """PAB decides on timesteps only: FP8 mode takes the same skip plan at each of 8 steps, and replays its caches."""
    from videosys_b200.core.pab import pab_mgr

    kernels_emul_fp8.emulate(monkeypatch)
    kw = dict(spatial_broadcast=True, spatial_threshold=[100, 930], spatial_range=2, temporal_broadcast=True,
              temporal_threshold=[100, 930], temporal_range=3, cross_broadcast=True, cross_threshold=[100, 930], cross_range=4)
    steps = [950.0, 900.0, 800.0, 700.0, 600.0, 500.0, 300.0, 50.0]
    plans = {}
    for fp8 in (False, True):
        net = _net().set_fp8_linears(fp8) if fp8 else _net()
        seen = []
        orig = net.pab_plan
        net.pab_plan = lambda ts, _o=orig, _s=seen: _s.append(_o(ts)) or _s[-1]
        pab_mgr.set_pab_manager(pab_mgr.PABConfig(**kw))
        pab_mgr.update_steps(len(steps))
        net.reset_pab_state()
        try:
            inp = cases.forward_inputs(BF)
            for t in steps:
                inp["timestep"] = torch.tensor([t, t])
                out = _run(net, inp)
                assert torch.isfinite(out).all()
        finally:
            pab_mgr.set_pab_manager(None)
        plans[fp8] = seen
    assert len(plans[True]) == len(steps) and plans[True] == plans[False]
    assert any(any(a or c for a, c in p) for p in plans[True])  # some step reuses a cache


def test_fp8_refuses_sequence_parallel(monkeypatch):
    kernels_emul_fp8.emulate(monkeypatch)
    net = _net(depth=1)
    net.parallel_manager = types.SimpleNamespace(sp_size=2, cp_size=1)
    with pytest.raises(NotImplementedError):
        net.set_fp8_linears(True)
    net.parallel_manager = None
    net.set_fp8_linears(True)
    net.parallel_manager = types.SimpleNamespace(sp_size=2, cp_size=1, sp_rank=0, sp_group=None)
    with pytest.raises(NotImplementedError):
        _run(net, cases.forward_inputs(BF))


def test_open_sora_config_fp8_default_off():
    from videosys_b200.pipelines.open_sora.pipeline_open_sora import OpenSoraConfig

    assert OpenSoraConfig().fp8_linears is False
    assert OpenSoraConfig(fp8_linears=True).fp8_linears is True
