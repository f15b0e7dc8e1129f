"""Open-Sora-Plan v1.2.0 conv down-sampler variants on the H100: the new kernels (vsb_dwconv_shuffle, vsb_dwconv_ffn,
vsb_gate_residual_unshuffle, the erf-GELU GEMM epilogue) against torch's eager ops on identical 16-bit inputs, and the model
against the outputs of the unmodified reference model (tests/golden/osp_v120_ds.pt)."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import osp_cases as OC, synth
from oracle.gen_golden_osp_ds import CASES12_DS, inputs_ds, weights_ds

pytestmark = pytest.mark.gpu
DTS = [torch.bfloat16, torch.float16]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _ulps(got, want):
    """Distance in units in the last place between two 16-bit tensors of the same sign pattern (bit patterns as integers)."""
    g, w = got.view(torch.int16).int(), want.view(torch.int16).int()
    g = torch.where(g < 0, -(g & 0x7FFF), g)
    w = torch.where(w < 0, -(w & 0x7FFF), w)
    return (g - w).abs()


def _assert_close_bits(got, want, what):
    d = _ulps(got, want)
    eq = (d == 0).float().mean().item()
    print(f"[parity] {what}: {100 * eq:.3f} % bit-equal, max {int(d.max())} ulp")
    assert eq >= 0.99 and int(d.max()) <= 1, what


def _rnd(tag, shape, dt, scale=1.0):
    return (synth.normalish(tag, shape) * scale).to(dt).cuda()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("B,T,H,W,C,ks,down", [(1, 4, 6, 10, 2304, (3, 3, 3), (2, 2, 2)),   # released width, edge tiles
                                                (2, 1, 30, 40, 2304, (1, 3, 3), (1, 2, 2)),  # 2-D variant, one frame
                                                (1, 2, 9, 7, 4608, (3, 5, 5), (1, 3, 7)),
                                                (2, 3, 5, 6, 64, (1, 5, 3), (3, 1, 2))])
def test_dwconv_shuffle_vs_eager(B, T, H, W, C, ks, down, dt):
    _need_gpu()
    from tests.kernels_emul_ds import unshuffle as _unshuffle
    from videosys_b200 import kernels as K

    x = _rnd(f"dws.x.{C}.{T}", (B, T * H * W, C), dt)
    w = _rnd(f"dws.w.{C}", (C, 1, *ks), dt, 0.3)
    b = _rnd(f"dws.b.{C}", (C,), dt, 0.3)
    taps = w.reshape(C, -1).t().contiguous()
    got = K.dwconv_shuffle(x, taps, b, B, T, H, W, ks, down)
    got2 = K.dwconv_shuffle(x, taps, b, B, T, H, W, ks, down)
    assert torch.equal(got, got2), "repeated launches differ"
    xi = x.view(B, T, H, W, C).permute(0, 4, 1, 2, 3)
    if ks[0] == 1:  # per frame, as DownSampler2d
        x2 = xi.transpose(1, 2).reshape(B * T, C, H, W)
        y = F.conv2d(x2, w.view(C, 1, ks[1], ks[2]), b, padding=(ks[1] // 2, ks[2] // 2), groups=C) + x2
        y = y.view(B, T, C, H, W).transpose(1, 2)
    else:
        y = F.conv3d(xi, w, b, padding=tuple(k // 2 for k in ks), groups=C) + xi
    want = y.permute(0, 2, 3, 4, 1).reshape(B, T * H * W, C)
    _assert_close_bits(_unshuffle(got, B, T, H, W, down), want, f"dwconv_shuffle {dt} {B}x{T}x{H}x{W}x{C} k{ks} s{down}")


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("BT,H,W,C", [(2, 6, 10, 4608), (16, 30, 40, 4608), (1, 1, 3, 128), (3, 9, 13, 384)])
def test_dwconv_ffn_vs_eager(BT, H, W, C, dt):
    _need_gpu()
    from videosys_b200 import kernels as K

    h = _rnd(f"dwf.h.{C}.{H}", (BT, H, W, C), dt)
    convs = [(_rnd(f"dwf.w{k}.{C}", (C, 1, k, k), dt, 0.3), _rnd(f"dwf.b{k}.{C}", (C,), dt, 0.3)) for k in (5, 3, 1)]
    taps = torch.cat([w.reshape(C, -1).t() for w, _ in convs], 0).contiguous()
    bias = torch.stack([b for _, b in convs], 0).contiguous()
    got = K.dwconv_ffn(h, taps, bias, BT, H, W)
    assert torch.equal(got, K.dwconv_ffn(h, taps, bias, BT, H, W)), "repeated launches differ"
    xi = h.permute(0, 3, 1, 2)
    out = xi
    for (w, b), k in zip(convs, (5, 3, 1)):  # FeedForward_Conv2d.forward: out = out + module(x)
        out = out + F.conv2d(xi, w, b, padding=k // 2, groups=C)
    _assert_close_bits(got, out.permute(0, 2, 3, 1), f"dwconv_ffn {dt} {BT}x{H}x{W}x{C}")


@pytest.mark.parametrize("dt", DTS)
def test_gate_residual_unshuffle_bit_exact(dt):
    _need_gpu()
    from tests.kernels_emul_ds import unshuffle as _unshuffle
    from videosys_b200 import kernels as K

    B, T, H, W, C, down = 2, 4, 6, 10, 2304, (2, 2, 2)
    x = _rnd("gru.x", (B, T * H * W, C), dt)
    y = _rnd("gru.y", (B * 8, T * H * W // 8, C), dt)
    mod = _rnd("gru.mod", (2, B, 6, C), dt)
    got = K.gate_residual_unshuffle(x, y, mod, 2, B, T, H, W, down)
    want = x + mod[0, :, 2].unsqueeze(1) * _unshuffle(y, B, T, H, W, down)
    assert torch.equal(got, want)
    x2 = x.clone()
    K.gate_residual_unshuffle(x2, y, mod, 2, B, T, H, W, down, out=x2)  # in place, as the model calls it
    assert torch.equal(x2, want)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("M,N,K_", [(9600, 4608, 2304), (77, 384, 192)])
def test_gemm_erf_gelu_epilogue_bit_exact(M, N, K_, dt):
    _need_gpu()
    from videosys_b200 import kernels as K

    a, w, b = _rnd(f"gelu.a.{M}", (M, K_), dt), _rnd(f"gelu.w.{N}", (N, K_), dt, 0.05), _rnd(f"gelu.b.{N}", (N,), dt)
    got = K.gemm_bias_act(a, w, b, act=2)
    assert torch.equal(got, F.gelu(K.gemm_bias_act(a, w, b, act=0)))
    assert torch.equal(got, K.gemm_bias_act(a, w, b, act=2))


# ---- the model against the unmodified reference ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "osp_v120_ds.pt"))


def _net(name, dt):
    from videosys_b200.models.transformers.open_sora_plan_v120_transformer_3d import OpenSoraT2V

    net = OpenSoraT2V(**CASES12_DS[name][0])
    net.load_state_dict(weights_ds(net.state_dict(), name, dt))
    return net.to(dt).to("cuda:0").eval()


@pytest.mark.parametrize("dt,dn", [(torch.bfloat16, "bf16"), (torch.float16, "fp16")])
@pytest.mark.parametrize("name", list(CASES12_DS))
def test_osp_v120_downsampler_forward_vs_reference_golden(gold, name, dt, dn):
    _need_gpu()
    from videosys_b200 import kernels

    net = _net(name, dt)
    x, enc, m, tt = inputs_ds(name, dt)
    n0 = kernels.launch_count()
    out = net(x.cuda(), timestep=tt.cuda(), encoder_hidden_states=enc.cuda(), encoder_attention_mask=m, return_dict=False)[0].cpu()
    launched = kernels.launch_count() - n0
    r32, r16 = gold[f"{name}.fp32"], gold[f"{name}.{dn}"]
    e_ours, e_ref = _rel(out, r32), _rel(r16, r32)
    print(f"[parity] osp v120 {name} {dn}: ours-vs-reference fp32 {e_ours:.3e}, reference {dn}-vs-fp32 {e_ref:.3e}, kernels {launched}")
    assert out.shape == r32.shape
    assert e_ours <= 1.25 * e_ref


def test_osp_v120_downsampler_pab_steps_vs_reference_golden(gold):
    _need_gpu()
    from videosys_b200 import kernels
    from videosys_b200.core.pab import pab_mgr

    dt = torch.bfloat16
    net = _net("ds3_rope", dt)
    pab_mgr.set_pab_manager(pab_mgr.PABConfig(**OC.PAB12_KW))
    pab_mgr.update_steps(len(OC.PAB_TIMESTEPS))
    net.reset_pab_state()
    try:
        launches = []
        for step, t in enumerate(OC.PAB_TIMESTEPS):
            x, enc, m, _ = inputs_ds("ds3_rope", dt, step)
            n0 = kernels.launch_count()
            out = net(x.cuda(), timestep=torch.tensor([t, t]).cuda(), encoder_hidden_states=enc.cuda(), encoder_attention_mask=m,
                      return_dict=False, ts_int=t)[0].cpu()
            launches.append(kernels.launch_count() - n0)
            r32, r16 = gold[f"pab.{step}.fp32"], gold[f"pab.{step}.bf16"]
            e_ours, e_ref = _rel(out, r32), _rel(r16, r32)
            print(f"[parity] osp v120 k333_s222 PAB step {step} t={t}: ours {e_ours:.3e}, reference bf16 {e_ref:.3e}, "
                  f"kernels {launches[-1]}")
            assert e_ours <= 1.25 * e_ref, step
        assert min(launches) < launches[0], launches
    finally:
        pab_mgr.set_pab_manager(None)


def test_osp_v120_downsampler_pipeline_generate():
    _need_gpu()
    from videosys_b200 import OpenSoraPlanConfig, VideoSysEngine

    tc = dict(CASES12_DS["ds3_rope"][0])
    kw = dict(num_inference_steps=4, guidance_scale=7.5, seed=0, max_sequence_length=24)
    eng = VideoSysEngine(OpenSoraPlanConfig(version="v120", transformer_type="29x480p", transformer_config=tc))
    try:
        out = eng.generate("Sunset over the sea.", **kw).video
        assert out.shape == (1, 4, 4, 8, 8) and torch.isfinite(out).all()
        assert torch.equal(eng.generate("Sunset over the sea.", **kw).video, out)
    finally:
        eng.shutdown()
