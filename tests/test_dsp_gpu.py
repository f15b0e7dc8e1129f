"""DSP on real GPUs (needs >= 2 devices; run with `python -m pytest tests/test_dsp_gpu.py -m gpu`).

  * the fused P2P switch (vsb_ln_modulate_dsp: the modulate kernel's stores are the switch; vsb_gate_residual_dsp: the
    gate + residual kernel pulls the branch from the peers) against the standalone modulate and gate + residual kernels
    composed with the oracle's index math, with padding on both axes, repeated (epoch / window reuse);
  * STDiT3 forward sharded over the ranks (fused P2P and NCCL transports) == the single-rank forward, bit for bit: the
    switch is a permutation and every kernel is row-independent; the same for 6 denoising steps through the replayed
    step graph (device-side epochs).
"""
import os
import traceback

import pytest
import torch
import torch.multiprocessing as mp

from oracle import cases, dsp_oracle, synth
from tests.helpers import stdit3_state_dict_template

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _need(n):
    if not torch.cuda.is_available() or torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")


def _worker(rank, world, port, q, transport):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        os.environ["VSB_DSP_P2P"] = "0" if transport == "nccl" else "1"
        import torch.distributed as dist

        from videosys_b200.core.distributed import comm
        from videosys_b200.core.distributed.parallel_mgr import ParallelManager, initialize
        from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config

        initialize(rank, world)
        dev = torch.device("cuda", rank)
        pm = ParallelManager(1, 1, world)
        res = {}
        if transport == "p2p":
            # the fused switch against the oracle's index math: push = modulate + S-shard -> T-shard, pull = T-shard ->
            # S-shard + gate + residual; padding on both axes; three rounds over the same windows and epoch counters
            from videosys_b200 import kernels as K

            for (B, T, S, C) in ((1, 5, 9, 64), (2, 4, 8, 64), (2, 20, 30, 288)):
                full = synth.normalish(f"fz{T}{S}", (B, T, S, C)).to(BF)
                shards = dsp_oracle.split_sequence(full, world, dim=2)
                Sl = shards[0].shape[2]
                xs = [s.to(dev).reshape(B, T * Sl, C) for s in shards]
                Tl = -(-(B * T) // world)
                p2p = comm.DspP2P(pm.sp_group, max(B * T * Sl, Tl * Sl * world) * C, dev)
                t6 = synth.normalish(f"fz.t{C}", (B, 6 * C), std=0.5).to(BF).to(dev)
                t06 = synth.normalish(f"fz.t0{C}", (B, 6 * C), std=0.5).to(BF).to(dev)
                tab = synth.normalish(f"fz.tab{C}", (6, C), std=0.3).to(BF).to(dev)
                mod = K.modulation_table(tab, t6, t06)
                xm_mask = torch.ones(B, T, dtype=torch.uint8, device=dev)
                xm_mask[0, 0] = 0
                x2 = xs[rank]
                wins, y = _fused_expected([K.ln_modulate(x, mod, xm_mask, 0, 1, B, T, Sl).cpu() for x in xs], B, T, S, rank)
                win = wins[rank].to(dev)
                cache_ref = torch.empty_like(x2)
                ref_b = K.gate_residual(x2, y.to(dev), mod, xm_mask, 2, B, T, Sl, cache_out=cache_ref)

                def fence():  # the test reuses the windows back to back, outside the block's own ordering
                    torch.cuda.synchronize()
                    dist.barrier()

                ok = []
                for rep in range(3):
                    got_a = p2p.ln_modulate_push(x2, mod, xm_mask, 0, 1, B, T, Sl, S).reshape(win.shape).clone()
                    fence()
                    p2p.branch_window(B, T, S, C).copy_(win.reshape(-1, C))
                    cache = torch.empty_like(x2)
                    got_b = p2p.gate_residual_pull(x2, mod, xm_mask, 2, B, T, Sl, S, cache_out=cache)
                    fence()
                    ok.append((torch.equal(got_a, win), torch.equal(got_b, ref_b), torch.equal(cache, cache_ref)))
                res[("fused", B, T, S)] = tuple(all(v) for v in zip(*ok))
                p2p.close()
        cfg = cases.small_model_cfg(depth=2)
        sd = synth.fill_state_dict(stdit3_state_dict_template(cfg, BF), "golden.")
        net = STDiT3(STDiT3Config(**cfg)).to(BF)
        net.load_state_dict(sd)
        net = net.to(dev).eval()
        net.enable_parallel(parallel_mgr=pm)
        inp = cases.forward_inputs(BF)
        gi = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in inp.items()}
        out = net(**gi)
        torch.cuda.synchronize()
        res["forward"] = out.cpu()
        res["steps"] = _four_steps(net, gi, dev, graph=True).cpu()
        q.put((rank, res, None))
        dist.barrier()
        dist.destroy_process_group()
    except Exception:
        q.put((rank, None, traceback.format_exc()))


def _fused_expected(outs, B, T, S, rank):
    """What the fused switch must deliver on `rank`, from the oracle's index math.  outs[r]: the modulate output of rank
    r's S-shard, [B, T*Sl, C] on the host.  The (batch, frame) sequences are what is scattered, so the oracle switches
    B*T sequences of one sample.  Returns every rank's T-shard window [1, Tl*S, C] (what ln_modulate_push leaves in it)
    and this rank's y [B, T*Sl, C] switched back from those windows (zero in the pad columns)."""
    C = outs[0].shape[-1]
    wins = dsp_oracle.dynamic_switch([o.reshape(1, -1, C) for o in outs], B * T, S, to_spatial_shard=False)[0]
    y = dsp_oracle.dynamic_switch(wins, B * T, S, to_spatial_shard=True)[0][rank]
    return wins, y.reshape(B, -1, C)


def _four_steps(net, gi, dev, graph):
    """6 denoising steps from a fixed latent (with graph=True: two eager, one capture + replay, three replays)."""
    from videosys_b200.core.graph_step import StepGraph

    st = StepGraph(net, 7.0, enabled=graph)
    fwd = {k: v for k, v in gi.items() if k not in ("x", "timestep")}
    z = gi["x"][:1].to(BF).contiguous()
    # step 1 eager (bf16 latent), step 2 eager (first sight of the fp32-latent key), step 3 captures, 4..6 replay
    for t in (900.0, 800.0, 700.0, 500.0, 300.0, 100.0):
        z = st.step(z, torch.tensor([t], device=dev), torch.tensor([0.1], device=dev), fwd)
    torch.cuda.synchronize()
    if graph:
        assert st.replays >= 3, st.replays
    del st  # the captured graphs hold NCCL work: release them before the process group goes away
    return z


def _single_rank_forward():
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config

    dev = torch.device("cuda:0")
    cfg = cases.small_model_cfg(depth=2)
    sd = synth.fill_state_dict(stdit3_state_dict_template(cfg, BF), "golden.")
    net = STDiT3(STDiT3Config(**cfg)).to(BF)
    net.load_state_dict(sd)
    net = net.to(dev).eval()
    inp = cases.forward_inputs(BF)
    gi = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in inp.items()}
    return net(**gi).cpu(), _four_steps(net, gi, dev, graph=False).cpu()


def _world():
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    return 8 if n >= 8 else (4 if n >= 4 else 2)


@pytest.mark.parametrize("transport", ["p2p", "nccl"])
def test_dsp_two_gpus(transport):
    """Runs on 2, 4 or 8 ranks (whatever the box has): reshard vs the oracle, and sharded forward == unsharded."""
    _need(2)
    world, port = _world(), 29800 + (os.getpid() % 100) + ["p2p", "nccl"].index(transport)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, transport), daemon=True) for r in range(world)]
    [p.start() for p in procs]
    got = {}
    try:
        for _ in range(world):
            r, res, err = q.get(timeout=240)
            assert err is None, err
            got[r] = res
        [p.join(timeout=60) for p in procs]
    finally:  # a rank that failed leaves its peers blocked in a collective: never leave them on the GPUs
        for p in procs:
            if p.is_alive():
                p.kill()
        [p.join(timeout=10) for p in procs]
    if transport == "p2p":
        for r in range(world):
            for k, v in got[r].items():
                if isinstance(k, tuple) and k[0] == "fused":
                    assert all(v), f"fused DSP kernels differ from the oracle: case {k[1:]} rank {r}: " \
                                   f"push {v[0]}, pull {v[1]}, pull cache {v[2]}"
    ref, ref_steps = _single_rank_forward()
    for r in range(world):
        assert torch.equal(got[r]["forward"], ref), f"sp={world} ({transport}) forward differs from sp=1 on rank {r}"
        assert torch.equal(got[r]["steps"], ref_steps), f"sp={world} ({transport}) 6 graph-replayed steps differ from sp=1 eager on rank {r}"
