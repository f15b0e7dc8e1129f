"""Open-Sora-Plan v1.1.0 with KV compression (``compress_kv_factor`` > 1): the front end's host logic on the torch stand-ins of
the kernels (tests/kernels_emul.py, tests/kernels_emul_kvc.py), fp32, against the outputs of the UNMODIFIED reference model
stored in tests/golden/osp_v110_kvc.pt (oracle/gen_golden_osp_kvc.py), the state-dict layout against the reference, the
configurations the reference cannot run, and frame-sharded sequence parallelism on two gloo ranks."""
import os

import pytest
import torch

from oracle import osp_cases as OC, ref_loader
from oracle.gen_golden_osp_kvc import CASES_KVC, PAB_CASE, inputs_kvc, weights_kvc
from tests import kernels_emul_kvc
from videosys_b200.models.transformers.open_sora_plan_v110_transformer_3d import LatteT2V


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "osp_v110_kvc.pt"))


def _net(name):
    net = LatteT2V(**CASES_KVC[name][0])
    net.load_state_dict(weights_kvc(net.state_dict(), name, torch.float32))
    return net.eval()


def _call(net, x, enc, m, t, all_ts=(900, 500), **kw):
    return net(x, timestep=t, all_timesteps=list(all_ts), encoder_hidden_states=enc, encoder_attention_mask=m, return_dict=False,
               **kw)[0]


@pytest.mark.parametrize("name", list(CASES_KVC))
def test_osp_v110_kv_compress_host_logic_vs_reference_golden(monkeypatch, gold, name):
    kernels_emul_kvc.emulate(monkeypatch)
    out = _call(_net(name), *inputs_kvc(name, torch.float32))
    if f"{name}.idx" in gold:
        assert list(out.shape) == gold[f"{name}.shape"]
        out = out.flatten()[gold[f"{name}.idx"].long()]
    want = gold[f"{name}.fp32"]
    assert out.shape == want.shape
    # the wide case sums 1152- and 4096-long fp32 dot products in another order than the reference's CPU kernels
    atol = 1e-4 * float(want.abs().max()) if name.startswith("wide") else 1e-5
    assert torch.allclose(out, want, rtol=1e-4, atol=atol), (out - want).abs().max()


def test_osp_v110_kv_compress_pab_steps_vs_reference_golden(monkeypatch, gold):
    """Eight PAB steps (spatial / temporal / cross broadcast and the MLP skip) with compressed blocks."""
    from videosys_b200.core.pab import pab_mgr

    kernels_emul_kvc.emulate(monkeypatch)
    net = _net(PAB_CASE)
    pab_mgr.set_pab_manager(pab_mgr.PABConfig(**OC.PAB_KW))
    pab_mgr.update_steps(len(OC.PAB_TIMESTEPS))
    net.reset_pab_state()
    try:
        for step, t in enumerate(OC.PAB_TIMESTEPS):
            x, enc, m, _ = inputs_kvc(PAB_CASE, torch.float32, step)
            out = _call(net, x, enc, m, torch.tensor([t, t]), OC.PAB_TIMESTEPS, ts_int=t)
            want = gold[f"pab.{step}.fp32"]
            assert torch.allclose(out, want, rtol=1e-4, atol=1e-5), (step, (out - want).abs().max())
    finally:
        pab_mgr.set_pab_manager(None)


@pytest.mark.parametrize("name", ["k2_f5", "k3_g7"])
def test_osp_v110_kv_compress_state_dict_matches_reference(name):
    if not ref_loader.available():
        pytest.skip("reference checkout not present")
    cfg = CASES_KVC[name][0]
    ref = ref_loader.build_osp_v110(dtype=torch.float32, **cfg)
    ours = LatteT2V(**cfg)
    rs, os_ = ref.state_dict(), ours.state_dict()
    assert {k: tuple(v.shape) for k, v in rs.items()} == {k: tuple(v.shape) for k, v in os_.items()}
    ours.load_state_dict(weights_kvc(rs, name, torch.float32), strict=True)
    ref.load_state_dict(ours.state_dict(), strict=True)


def test_osp_v110_kv_compress_layers_only_in_second_half():
    """sr / norm exist in blocks d >= num_layers // 2 of both stacks (reference :2283-2320), with the reference's shapes and
    initial values (:1101-1122); an uncompressed model has none."""
    C, k = 144, 2
    cfg = dict(CASES_KVC["k2_f5"][0], num_layers=4)
    net = LatteT2V(**cfg)
    sd = net.state_dict()
    for d in range(4):
        for stack in ("transformer_blocks", "temporal_transformer_blocks"):
            assert (f"{stack}.{d}.attn1.sr.weight" in sd) == (d >= 2)
    assert tuple(sd["transformer_blocks.2.attn1.sr.weight"].shape) == (C, 1, k, k)
    assert tuple(sd["temporal_transformer_blocks.3.attn1.sr.weight"].shape) == (C, 1, k)
    assert tuple(sd["temporal_transformer_blocks.3.attn1.norm.bias"].shape) == (C,)
    assert torch.all(sd["transformer_blocks.2.attn1.sr.weight"] == 0.25) and torch.all(sd["transformer_blocks.2.attn1.sr.bias"] == 0)
    assert torch.all(sd["temporal_transformer_blocks.2.attn1.sr.weight"] == 0.5)
    assert net.transformer_blocks[2].attn1.norm.eps == 1e-5
    plain = LatteT2V(**dict(cfg, compress_kv_factor=1)).state_dict()
    assert not any(".sr." in n or ".attn1.norm." in n for n in plain)


def test_osp_v110_kv_compress_rejections(monkeypatch):
    kernels_emul_kvc.emulate(monkeypatch)
    base = CASES_KVC["k2_f5"][0]
    with pytest.raises(ValueError, match="RoPE"):  # reference :2200
        LatteT2V(**dict(base, use_rope=True))
    for bad in (0, 1.5):
        with pytest.raises(ValueError, match="positive integer"):
            LatteT2V(**dict(base, compress_kv_factor=bad))
    _, _, L, _ = CASES_KVC["k2_f5"]
    enc, m, t = torch.zeros(2, 1, L, 32), torch.ones(2, 1, L), torch.tensor([500, 500])
    with pytest.raises(ValueError, match="4x4 patches"):  # k = 5
        _call(LatteT2V(**dict(base, compress_kv_factor=5)).eval(), torch.zeros(2, 4, 5, 8, 8), enc, m, t)
    with pytest.raises(ValueError, match="1x4 patches"):  # k = 2
        _call(LatteT2V(**dict(base, sample_size=(2, 8))).eval(), torch.zeros(2, 4, 5, 2, 8), enc, m, t)
    with pytest.raises(ValueError, match="3x3 patches and 2 frames"):  # k = 3; an even frame count gets no padding
        _call(LatteT2V(**dict(base, sample_size=(6, 6), video_length=2, compress_kv_factor=3)).eval(), torch.zeros(2, 4, 2, 6, 6),
              enc, m, t)


def _sp_worker(rank, world, port, name, q):
    import traceback

    os.environ["CUDA_VISIBLE_DEVICES"] = ""  # a CPU test: gloo ranks, never NCCL on a shared local GPU
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        import torch.distributed as dist

        from videosys_b200.core.distributed.parallel_mgr import initialize

        kernels_emul_kvc.emulate_global()
        initialize(rank, world)
        net = _net(name)
        args = inputs_kvc(name, torch.float32)
        want = _call(net, *args)  # unsharded (parallel_manager None)
        net.enable_parallel(1, world, False)
        got = _call(net, *args)
        q.put((rank, float((got - want).abs().max()), float(want.abs().max()), tuple(got.shape) == tuple(want.shape), None))
        dist.barrier()
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        q.put((rank, None, None, None, traceback.format_exc()))


@pytest.mark.parametrize("name", ["k2_f5", "k2_f4"])
def test_osp_v110_kv_compress_sequence_parallel_gloo_world2(name):
    """Two ranks, frame-sharded DSP: the spatial compression runs on each rank's frames, the temporal one after the switch to
    the patch shard (every frame present, the odd-count padding included); both ranks reproduce the single-rank forward."""
    import multiprocessing as mp

    world, port = 2, 31400 + (os.getpid() % 300) + 3 * list(CASES_KVC).index(name)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sp_worker, args=(r, world, port, name, q)) for r in range(world)]
    [p.start() for p in procs]
    for _ in range(world):
        r, err_abs, scale, same_shape, tb = q.get(timeout=300)
        assert tb is None, tb
        assert same_shape and err_abs <= 1e-4 * max(scale, 1.0), (name, r, err_abs, scale)
    [p.join(timeout=60) for p in procs]
