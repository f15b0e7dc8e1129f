"""OpenSora v1.2 denoising steps with the FP8 Linears off and on (STDiT3.set_fp8_linears), in one process.

The workload is bench.py's (random-init STDiT3 at the full 28-block size, synthetic caption and latent, CFG pair), with
every kernel launched from the host (no step graphs, so the two modes share no captured memory pool): ``--steps`` timed steps per mode after ``--warmup`` steps, the two modes alternating for ``--rounds``
rounds from the same latent; the median ms per step of each mode is reported.  A separate untimed eager step per mode
splits the device time by kernel kind (gemm, gemm_fp8, quant, attn, rest) with CUDA events.  The relative L2 distance
between the two modes' latents after the timed steps of the first round is the quality proxy: with random weights it
says how far the quantization moves a step, not what it does to a video.  ``--pab`` runs the steps inside PAB's
broadcast range (schedule index 22 on), as bench.py does.  Prints one JSON line; writes nothing unless --out is given.

    python bench_fp8.py [--workload opensora_720p_68f_50step] [--steps 4] [--warmup 3] [--rounds 3] [--pab] [--out F]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

KINDS = {"gemm": "gemm", "gemm_fp8": "gemm_fp8", "quant": "quant", "attn_flash": "attn", "attn_short": "attn"}


def main():
    import bench
    from bench_gemm import gpu_info
    from videosys_b200 import kernels
    from videosys_b200.core.graph_step import StepGraph
    from videosys_b200.core.pab import pab_mgr
    from videosys_b200.models.transformers.open_sora_transformer_3d import STDiT3, STDiT3Config
    from videosys_b200.pipelines.open_sora.pipeline_open_sora import OpenSoraPABConfig
    from videosys_b200.schedulers.scheduling_rflow_open_sora import RFLOW

    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="opensora_720p_68f_50step", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pab", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8.py needs a CUDA device")
    dev, bf = torch.device("cuda", 0), torch.bfloat16
    W = bench.WORKLOADS[a.workload]
    torch.manual_seed(0)
    net = STDiT3(STDiT3Config(**bench.MODEL)).to(bf).to(dev).eval()
    sched = RFLOW(num_sampling_steps=W["steps"], cfg_scale=7.0, use_timestep_transform=True)
    T, Hl, Wl = W["lat"]
    g = torch.Generator(device="cpu").manual_seed(1)
    z0 = torch.randn(1, 4, T, Hl, Wl, generator=g).to(dev, bf)
    y = torch.randn(1, 1, W["L"], bench.MODEL["caption_channels"], generator=g).to(dev, bf)
    y_null = net.y_embedder.y_embedding[None, None].to(bf)
    margs = dict(y=torch.cat([y, y_null], 0), mask=torch.ones(1, W["L"], dtype=torch.long, device=dev),
                 height=torch.tensor([W["h"]], device=dev, dtype=bf), width=torch.tensor([W["w"]], device=dev, dtype=bf),
                 num_frames=torch.tensor([W["frames"]], device=dev, dtype=bf), fps=torch.tensor([24], device=dev, dtype=bf))
    ts_cpu = sched.prepare_timesteps(1, "cpu", {k: v.cpu() for k, v in margs.items() if k in ("height", "width", "num_frames")})
    timesteps = [t.to(dev) for t in ts_cpu]
    ts_int = [int(t.to(bf).item()) for t in ts_cpu]
    n_ts = len(timesteps)
    dts = [((timesteps[i] - timesteps[i + 1] if i < n_ts - 1 else timesteps[i]) / 1000.0) for i in range(n_ts)]
    fwd = {k: v for k, v in margs.items() if k != "num_frames"}
    fwd["x_mask"] = torch.ones(2, T, dtype=torch.bool, device=dev)
    first = 22 if a.pab else 0

    def pab_reset():
        pab_mgr.set_pab_manager(OpenSoraPABConfig() if a.pab else None)
        if a.pab:
            pab_mgr.update_steps(W["steps"])
        net.reset_pab_state()

    stepper = StepGraph(net, 7.0, enabled=False)

    def run(mode, n):
        net.set_fp8_linears(mode)
        pab_reset()
        z = z0.clone()
        for i in range(n):
            k = (first + i) % n_ts
            z = stepper.step(z, timesteps[k], dts[k], fwd, ts_int=ts_int[k])
        return z

    for mode in (False, True):  # warm-up
        run(mode, a.warmup)
    ms = {False: [], True: []}
    lat = {}
    for r in range(a.rounds):
        for mode in (False, True):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            z = run(mode, a.steps)
            e1.record()
            torch.cuda.synchronize()
            ms[mode].append(e0.elapsed_time(e1) / a.steps)
            if r == 0:
                lat[mode] = z.double()
            print(f"round {r} fp8={mode}: {ms[mode][-1]:.2f} ms/step", flush=True)
    rel = ((lat[True] - lat[False]).norm() / lat[False].norm()).item()

    split = {}
    for mode in (False, True):  # kind split: one eager step, every launch between CUDA events
        net.set_fp8_linears(mode)
        pab_reset()
        kernels.PROFILE, kernels.PROFILE_KINDS = [], None
        stepper.step(z0.clone(), timesteps[first], dts[first], fwd, ts_int=ts_int[first])
        torch.cuda.synchronize()
        acc = {}
        for kind, s, e, _ in kernels.PROFILE:
            k = KINDS.get(kind, "rest")
            acc[k] = acc.get(k, 0.0) + s.elapsed_time(e)
        kernels.PROFILE = None
        split["fp8" if mode else "bf16"] = {k: round(v, 2) for k, v in sorted(acc.items())}
    net.set_fp8_linears(False)
    pab_mgr.set_pab_manager(None)
    res = dict(gpu=gpu_info(), workload=a.workload, pab=a.pab, steps=a.steps, rounds=a.rounds,
               ms_per_step_bf16=round(statistics.median(ms[False]), 2), ms_per_step_fp8=round(statistics.median(ms[True]), 2),
               speedup=round(statistics.median(ms[False]) / statistics.median(ms[True]), 3), latent_rel_l2=rel,
               eager_step_ms_by_kind=split)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
