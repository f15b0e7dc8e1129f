"""Times ``kernels.attn_flash`` alone at the shapes the model front ends hand it, one shape at a time:

  spatial_720p   OpenSora v1.2 720p spatial self-attention: 40 frames (CFG pair x 20) x 3600 tokens, 16 heads x 72,
                 q / k / v strided views of the packed qkv projection
  cross_720p     its text cross-attention: 72 000 queries per sample x 300 keys, k / v views of the packed kv (stride 2C)
  spatial_240p   OpenSora v1.2 240p spatial self-attention: 30 frames x 405 tokens
  temporal_30f   temporal self-attention at 30 frames (the flash path, T >= 30): batch = 3600 patches, row = frame,
                 written straight into the token-major output (strided output view)
  cogvideox_2b   CogVideoX-2B joint text + video attention, fp16: CFG pair x 17 776 tokens, 30 heads x 64
  vchitect_2b    Vchitect-2.0-2B spatial joint attention, bf16: 40 frames x (540 patches + 333 text tokens), 24 heads x 64

    python bench_attention.py [--iters 20] [--warmup 3] [--rounds 1] [--shapes a,b] [--out FILE.json]

Inputs are seeded (standard normal), so two builds given the same arguments can be compared output for output: every shape
prints the SHA-256 of its output bytes.  Rates are 4 nb H nq nk D FLOPs (Q K^T and P V) over the kernel time from CUDA
events around --iters back-to-back launches.  The card's name, power limit and SM clock (sampled while the launches run)
are part of the result.  Writes nothing unless --out is given.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# name: (nb, nq, nk, H, D, dtype, layout)
SHAPES = {
    "spatial_720p": (40, 3600, 3600, 16, 72, torch.bfloat16, "packed"),
    "cross_720p": (2, 72000, 300, 16, 72, torch.bfloat16, "cross"),
    "spatial_240p": (30, 405, 405, 16, 72, torch.bfloat16, "packed"),
    "temporal_30f": (3600, 30, 30, 16, 72, torch.bfloat16, "temporal"),
    "cogvideox_2b": (2, 17776, 17776, 30, 64, torch.float16, "packed"),
    "vchitect_2b": (40, 873, 873, 24, 64, torch.bfloat16, "packed"),
}


def make_call(name, dev, seed):
    """Seeded inputs of one shape; returns (launch(), output tensor, FLOPs per launch)."""
    from videosys_b200 import kernels

    nb, nq, nk, H, D, dt, layout = SHAPES[name]
    C = H * D
    g = torch.Generator(device=dev).manual_seed(seed)

    def rnd(*shape):
        return torch.randn(*shape, device=dev, generator=g).to(dt)

    scale = D**-0.5
    if layout == "packed":  # packed_self_attention: [nb * n, 3, C]
        q3 = rnd(nb * nq, 3, C)
        out = torch.empty(nb, nq, C, device=dev, dtype=dt)

        def launch():
            kernels.attn_flash(q3[:, 0], q3[:, 1], q3[:, 2], nb, nq, nk, H, D, 3 * C, nq * 3 * C, 3 * C, nq * 3 * C, scale, out=out)
    elif layout == "cross":  # cross_attention: q [nb * nq, C], kv [nb * nk, 2, C]
        q, kv = rnd(nb * nq, C), rnd(nb * nk, 2, C)
        out = torch.empty(nb, nq, C, device=dev, dtype=dt)

        def launch():
            kernels.attn_flash(q, kv[:, 0], kv[:, 1], nb, nq, nk, H, D, C, nq * C, 2 * C, nk * 2 * C, scale, out=out)
    else:  # temporal_attention, one sample: token-major [T, S, 3, C] -> out [T * S, C]; batch = patch, row = frame
        S, T = nb, nq
        q3 = rnd(T * S, 3, C)
        out = torch.empty(T * S, C, device=dev, dtype=dt)

        def launch():
            kernels.attn_flash(q3[:, 0], q3[:, 1], q3[:, 2], S, T, T, H, D, S * 3 * C, 3 * C, S * 3 * C, 3 * C, scale, out=out,
                               out_row_stride=S * C, out_batch_stride=C)
    return launch, out, 4 * nb * H * nq * nk * D


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def run_shape(name, seed, iters, warmup):
    from bench import ClockSampler

    launch, out, flops = make_call(name, "cuda" if torch.cuda.is_available() else "cpu", seed)
    if not torch.cuda.is_available():
        raise SystemExit(f"{name}: inputs built; timing needs a CUDA device")
    for _ in range(warmup):
        launch()
    torch.cuda.synchronize()
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        launch()
    e1.record()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    ms = e0.elapsed_time(e1) / iters
    digest = hashlib.sha256(out.view(torch.int16).cpu().numpy().tobytes()).hexdigest()
    del launch, out
    torch.cuda.empty_cache()
    return dict(ms=round(ms, 4), tflops=round(flops / (ms * 1e-3) / 1e12, 1), sha256=digest, sm_mhz=clocks["sm_mhz"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=1, help="time every shape this many times (in turn)")
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated subset of " + ", ".join(SHAPES))
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    names = [s for s in a.shapes.split(",") if s]
    bad = [s for s in names if s not in SHAPES]
    if bad:
        ap.error(f"unknown shapes {bad}")
    res = dict(gpu=gpu_info() if torch.cuda.is_available() else None, iters=a.iters, shapes={})
    for r in range(a.rounds):
        for i, name in enumerate(names):
            m = run_shape(name, a.seed + i, a.iters, a.warmup)
            print(f"round {r} {name:14s} {m['ms']:9.3f} ms {m['tflops']:7.1f} TFLOP/s  sm {m['sm_mhz']} MHz  sha256 {m['sha256']}",
                  flush=True)
            res["shapes"].setdefault(name, []).append(m)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
