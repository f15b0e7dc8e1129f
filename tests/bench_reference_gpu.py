#!/usr/bin/env python
"""R-GPU-1 (BASELINE.md section 2): the reference's eager PyTorch path on ONE GPU, i.e. the oracle's op-for-op
restatement of STDiT3.forward executed with torch/cuBLAS/SDPA library kernels on the GPU.  Measurement
infrastructure (lives under tests/ because it executes oracle/); never used by the product or by bench.py's value.

    python tests/bench_reference_gpu.py [--workload opensora_720p_68f_50step] [--steps 2]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import MODEL, WORKLOADS  # noqa: E402
from oracle import stdit3_oracle as O  # noqa: E402
from tests.helpers import stdit3_state_dict_template  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="opensora_720p_68f_50step")
    ap.add_argument("--steps", type=int, default=2)
    args = ap.parse_args()
    W = WORKLOADS[args.workload]
    dev = torch.device("cuda:0")
    bf = torch.bfloat16
    torch.manual_seed(0)
    cfg = dict(MODEL)
    sd = {}
    for k, v in stdit3_state_dict_template(cfg, bf).items():
        if k.endswith("rope.freqs"):
            sd[k] = O.rope_freqs(cfg["hidden_size"] // cfg["num_heads"]).to(bf).to(dev)
        elif v.ndim >= 2:
            sd[k] = (torch.randn(v.shape) * 0.02).to(bf).to(dev)
        else:
            sd[k] = (torch.randn(v.shape) * 0.02 + (1.0 if "norm" in k else 0.0)).to(bf).to(dev)
    T, Hl, Wl = W["lat"]
    z = torch.randn(2, 4, T, Hl, Wl, device=dev, dtype=bf)
    inp = dict(
        x=z, timestep=torch.tensor([900.0, 900.0], device=dev),
        y=torch.randn(2, 1, W["L"], MODEL["caption_channels"], device=dev, dtype=bf),
        mask=torch.ones(1, W["L"], dtype=torch.long, device=dev), x_mask=torch.ones(2, T, dtype=torch.bool, device=dev),
        fps=torch.tensor([24.0, 24.0], device=dev, dtype=bf), height=torch.tensor([float(W["h"])] * 2, device=dev, dtype=bf),
        width=torch.tensor([float(W["w"])] * 2, device=dev, dtype=bf),
    )
    ocfg = dict(hidden_size=cfg["hidden_size"], num_heads=cfg["num_heads"], depth=cfg["depth"])
    with torch.no_grad():
        O.stdit3_forward(sd, ocfg, **inp)  # warm-up
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            O.stdit3_forward(sd, ocfg, **inp)
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    out = {"what": "reference eager path (oracle restatement on torch/cuBLAS/SDPA), 1 GPU", "workload": args.workload,
           "ms_per_step": ms, "frames_per_s": W["frames"] / (W["steps"] * ms / 1e3), "steps_timed": args.steps,
           "torch": torch.__version__}
    print(json.dumps(out))
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "gpurun_out", f"ref_gpu_{args.workload}.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
