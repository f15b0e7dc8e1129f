"""Open-Sora-Plan v1.1.0 KV compression on the H100: ``vsb_kv_compress`` against torch's eager ops laid out the way the
reference calls them, the model against the outputs of the unmodified reference model (tests/golden/osp_v110_kvc.pt), the
public pipeline, and frame-sharded sequence parallelism on two GPUs."""
import os
import traceback

import pytest
import torch
import torch.multiprocessing as mp
import torch.nn.functional as F

from oracle import osp_cases as OC, synth
from oracle.gen_golden_osp_kvc import CASES_KVC, PAB_CASE, inputs_kvc, weights_kvc

pytestmark = pytest.mark.gpu
DTS = [torch.bfloat16, torch.float16]


def _need_gpus(n=1):
    if not torch.cuda.is_available() or torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} CUDA device(s)")


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _ulps(got, want):
    """Distance in units in the last place between two 16-bit tensors (bit patterns as sign-magnitude integers)."""
    g, w = got.view(torch.int16).int(), want.view(torch.int16).int()
    g = torch.where(g < 0, -(g & 0x7FFF), g)
    w = torch.where(w < 0, -(w & 0x7FFF), w)
    return (g - w).abs()


def _assert_close_ln(got, want, ng, what):
    """The down-sampler tests' criterion (>= 99 % bit-equal, <= 1 ulp), where one ulp is taken at max(|want|, |ng|), ng =
    |gamma * normalised| in fp32: where the LayerNorm's bias cancels that term, the output is much smaller than the operands
    of its last fma, and the fp32 statistics (summed in another order than torch's Welford) move it by up to one ulp of
    the operands, many ulps of the result."""
    d = _ulps(got, want)
    eq = (d == 0).float().mean().item()
    mant = 7 if got.dtype == torch.bfloat16 else 10
    scale = torch.maximum(want.float().abs(), ng)
    ulp = torch.exp2(torch.floor(torch.log2(scale.clamp_min(1e-30))) - mant)
    err = ((got.float() - want.float()).abs() / ulp).max().item()
    print(f"[parity] {what}: {100 * eq:.3f} % bit-equal, max {int(d.max())} ulp of the result, {err:.2f} ulp of max(|out|, |g*n|)")
    assert eq >= 0.99 and err <= 1.0, what


def _rnd(tag, shape, dt, scale=1.0, shift=0.0):
    return (synth.normalish(tag, shape) * scale + shift).to(dt).cuda()


def _layers(tag, C, taps_shape, dt):
    w = _rnd(tag + ".w", (C, 1, *taps_shape), dt, 0.3)
    return w, _rnd(tag + ".b", (C,), dt, 0.3), _rnd(tag + ".g", (C,), dt, 0.2, 1.0), _rnd(tag + ".beta", (C,), dt, 0.2)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("B,F_,h,w,C,k", [(2, 17, 32, 32, 1152, 2),  # 65x512x512: 1024 -> 256 keys per frame
                                          (1, 3, 31, 33, 1152, 2),   # odd grid: the last row / column is not read
                                          (2, 2, 7, 7, 1152, 3),     # k = 3, floors
                                          (1, 2, 4, 6, 64, 2)])
def test_kv_compress_spatial_vs_eager(B, F_, h, w, C, k, dt):
    """Conv2d(groups=C, stride=k) on the reference's channels-last view of the tokens (:1184-1186), then LayerNorm."""
    _need_gpus()
    from videosys_b200 import kernels as K

    x = _rnd(f"kvcs.x.{C}.{h}", (B, F_, h, w, C), dt)
    sw, sb, g, beta = _layers(f"kvcs.{C}.{k}", C, (k, k), dt)
    taps = sw.reshape(C, -1).t().contiguous()
    got = K.kv_compress(x, taps, sb, g, beta, B, F_, h, w, (1, k, k), 0, 1e-5, round_conv=True)
    assert torch.equal(got, K.kv_compress(x, taps, sb, g, beta, B, F_, h, w, (1, k, k), 0, 1e-5, round_conv=True)), \
        "repeated launches differ"
    hs = x.view(B * F_, h * w, C)
    e = F.conv2d(hs.permute(0, 2, 1).reshape(B * F_, C, h, w), sw, sb, stride=k, groups=C).reshape(B * F_, C, -1).permute(0, 2, 1)
    want = F.layer_norm(e, (C,), g, beta, 1e-5)
    ng = (F.layer_norm(e.float(), (C,), None, None, 1e-5) * g.float()).abs()
    _assert_close_ln(got.view(B * F_, -1, C), want, ng, f"kv_compress spatial {dt} {B}x{F_}x{h}x{w}x{C} k{k}")


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("B,F_,S,C,k", [(2, 17, 1024, 1152, 2),  # 65 frames: 17 (+1 copy of frame 0) -> 9 keys
                                        (1, 56, 256, 1152, 2),   # 221 frames: 56 -> 28, no padding
                                        (2, 17, 64, 1152, 3),    # k = 3: 17 + 2 -> 6
                                        (1, 5, 12, 64, 2)])
def test_kv_compress_temporal_vs_eager(B, F_, S, C, k, dt):
    """Conv1d(groups=C, stride=k) over the frames of each patch after k - 1 copies of frame 0 when the count is odd
    (:1188-1193), then LayerNorm."""
    _need_gpus()
    from videosys_b200 import kernels as K

    pad = k - 1 if F_ % 2 else 0
    x = _rnd(f"kvct.x.{C}.{S}", (B, F_, S, C), dt)
    sw, sb, g, beta = _layers(f"kvct.{C}.{k}", C, (k,), dt)
    taps = sw.reshape(C, -1).t().contiguous()
    got = K.kv_compress(x, taps, sb, g, beta, B, F_, S, 1, (k, 1, 1), pad, 1e-5, round_conv=False)
    assert torch.equal(got, K.kv_compress(x, taps, sb, g, beta, B, F_, S, 1, (k, 1, 1), pad, 1e-5, round_conv=False)), \
        "repeated launches differ"
    e = x.permute(0, 2, 1, 3).reshape(B * S, F_, C).permute(0, 2, 1)  # the temporal block's [(b s), f, C], channels first
    if pad:
        e = torch.cat((e[:, :, :1].repeat(1, 1, pad), e), dim=2)
    e = F.conv1d(e, sw, sb, stride=k, groups=C).permute(0, 2, 1)
    want = F.layer_norm(e, (C,), g, beta, 1e-5)
    ng = (F.layer_norm(e.float(), (C,), None, None, 1e-5) * g.float()).abs()
    _assert_close_ln(got.view(B, -1, S, C).permute(0, 2, 1, 3).reshape(B * S, -1, C), want, ng,
                     f"kv_compress temporal {dt} {B}x{F_}x{S}x{C} k{k} pad {pad}")


def test_kv_compress_rejects_bad_shapes():
    _need_gpus()
    from videosys_b200 import _lib, kernels as K

    C = 64
    x = torch.zeros(1, 2, 4, 4, C, dtype=torch.bfloat16, device="cuda")
    p = torch.zeros(4, C, dtype=torch.bfloat16, device="cuda")
    v = torch.zeros(C, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(_lib.VsbError, match="empty output grid"):
        K.kv_compress(x, p, v, v, v, 1, 2, 4, 4, (3, 1, 1), 0)
    with pytest.raises(_lib.VsbError, match="empty output grid"):
        K.kv_compress(x, p, v, v, v, 1, 2, 4, 4, (1, 5, 5), 0)
    x12 = torch.zeros(1, 2, 4, 4, 12, dtype=torch.bfloat16, device="cuda")
    v12 = torch.zeros(12, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(_lib.VsbError, match="C % 8"):
        K.kv_compress(x12, torch.zeros(4, 12, dtype=torch.bfloat16, device="cuda"), v12, v12, v12, 1, 2, 4, 4, (1, 2, 2), 0)


# ---- the model against the unmodified reference ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "osp_v110_kvc.pt"))


def _net(name, dt, dev="cuda:0"):
    from videosys_b200.models.transformers.open_sora_plan_v110_transformer_3d import LatteT2V

    net = LatteT2V(**CASES_KVC[name][0])
    net.load_state_dict(weights_kvc(net.state_dict(), name, dt))
    return net.to(dt).to(dev).eval()


def _call(net, x, enc, m, t, all_ts=(900, 500), dev="cuda:0", **kw):
    return net(x.to(dev), timestep=t.to(dev), all_timesteps=list(all_ts), encoder_hidden_states=enc.to(dev), encoder_attention_mask=m,
               return_dict=False, **kw)[0]


@pytest.mark.parametrize("dt,dn", [(torch.bfloat16, "bf16"), (torch.float16, "fp16")])
@pytest.mark.parametrize("name", list(CASES_KVC))
def test_osp_v110_kv_compress_forward_vs_reference_golden(gold, name, dt, dn):
    _need_gpus()
    from videosys_b200 import kernels

    net = _net(name, dt)
    n0 = kernels.launch_count()
    out = _call(net, *inputs_kvc(name, dt)).cpu()
    launched = kernels.launch_count() - n0
    if f"{name}.idx" in gold:
        assert list(out.shape) == gold[f"{name}.shape"]
        out = out.flatten()[gold[f"{name}.idx"].long()]
    r32, r16 = gold[f"{name}.fp32"], gold[f"{name}.{dn}"]
    e_ours, e_ref = _rel(out, r32), _rel(r16, r32)
    print(f"[parity] osp v110 kvc {name} {dn}: ours-vs-reference fp32 {e_ours:.3e}, reference {dn}-vs-fp32 {e_ref:.3e}, "
          f"kernels {launched}")
    assert out.shape == r32.shape
    assert e_ours <= 1.25 * e_ref


def test_osp_v110_kv_compress_pab_steps_vs_reference_golden(gold):
    _need_gpus()
    from videosys_b200 import kernels
    from videosys_b200.core.pab import pab_mgr

    dt = torch.bfloat16
    net = _net(PAB_CASE, dt)
    pab_mgr.set_pab_manager(pab_mgr.PABConfig(**OC.PAB_KW))
    pab_mgr.update_steps(len(OC.PAB_TIMESTEPS))
    net.reset_pab_state()
    try:
        launches = []
        for step, t in enumerate(OC.PAB_TIMESTEPS):
            x, enc, m, _ = inputs_kvc(PAB_CASE, dt, step)
            n0 = kernels.launch_count()
            out = _call(net, x, enc, m, torch.tensor([t, t]), OC.PAB_TIMESTEPS, ts_int=t).cpu()
            launches.append(kernels.launch_count() - n0)
            r32, r16 = gold[f"pab.{step}.fp32"], gold[f"pab.{step}.bf16"]
            e_ours, e_ref = _rel(out, r32), _rel(r16, r32)
            print(f"[parity] osp v110 kvc PAB step {step} t={t}: ours {e_ours:.3e}, reference bf16 {e_ref:.3e}, kernels {launches[-1]}")
            assert e_ours <= 1.25 * e_ref, step
        assert min(launches) < launches[0], launches
    finally:
        pab_mgr.set_pab_manager(None)


def test_osp_v110_kv_compress_pipeline_generate():
    _need_gpus()
    from videosys_b200 import OpenSoraPlanConfig, VideoSysEngine

    tc = dict(CASES_KVC["k2_f5"][0])
    assert tc["compress_kv_factor"] == 2 and tc["use_rope"] is False
    kw = dict(num_inference_steps=4, guidance_scale=7.5, seed=0, height=64, width=64, max_sequence_length=24)
    eng = VideoSysEngine(OpenSoraPlanConfig(version="v110", transformer_type="65x512x512", transformer_config=tc))
    try:
        out = eng.generate("Sunset over the sea.", **kw).video
        assert out.shape == (1, 4, 5, 8, 8) and torch.isfinite(out).all()
        assert torch.equal(eng.generate("Sunset over the sea.", **kw).video, out)
    finally:
        eng.shutdown()


# ---- two GPUs: frame-sharded DSP == one GPU ---------------------------------------------------------------------------------------
def _sp_run(dev, sp):
    res = {}
    for name in ("k2_f5", "k2_f4"):
        net = _net(name, torch.float16, dev)
        if sp:
            net.enable_parallel(1, 2, False)
        res[name] = _call(net, *inputs_kvc(name, torch.float16), dev=dev).cpu()
    torch.cuda.synchronize(dev)
    return res


def _worker(rank, world, port, q):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        import torch.distributed as dist

        from videosys_b200.core.distributed.parallel_mgr import initialize

        initialize(rank, world)
        q.put((rank, _sp_run(torch.device("cuda", rank), True), None))
        dist.barrier()
        dist.destroy_process_group()
    except Exception:
        q.put((rank, None, traceback.format_exc()))


def test_osp_v110_kv_compress_two_gpus():
    """Both ranks of sp = 2 (odd and even frame counts) reproduce the single-GPU forward bit for bit: the spatial compression
    is frame-local, the temporal one runs on the patch shard, which holds every frame."""
    _need_gpus(2)
    world, port = 2, 29700 + (os.getpid() % 80)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q), daemon=True) for r in range(world)]
    [p.start() for p in procs]
    got = {}
    try:
        for _ in range(world):
            r, res, err = q.get(timeout=300)
            assert err is None, err
            got[r] = res
        [p.join(timeout=60) for p in procs]
    finally:  # a rank that failed leaves its peer blocked in a collective: never leave it on the GPU
        for p in procs:
            if p.is_alive():
                p.kill()
        [p.join(timeout=10) for p in procs]
    ref = _sp_run(torch.device("cuda:0"), False)
    for r in range(world):
        for k, v in ref.items():
            assert torch.isfinite(v.float()).all(), k
            assert torch.equal(got[r][k], v), (k, r, (got[r][k].float() - v.float()).abs().max().item())
