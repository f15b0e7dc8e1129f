"""Measures Open-Sora-Plan v1.1.0's KV compression (compress_kv_factor = 2) at the 65x512x512 shape on one GPU:

  - time and achieved HBM bandwidth of vsb_kv_compress, spatial (2 x 2 window over the 32 x 32 patches of every frame) and
    temporal (2 frames per patch, 17 + 1 padded frames), from the bytes the algorithm must move (read the input once, write
    the output once) against the H100 SXM data-sheet 3.35 TB/s, next to the reference's eager chain (conv, LayerNorm);
  - ms per full-depth (28-layer) transformer step with compress_kv_factor 1 and 2 (both without RoPE, which compression
    excludes), timed in alternating rounds so that both see the same machine state.

    python bench_osp_kv_compress.py [--steps 10] [--warmup 3] [--rounds 3] [--out FILE.json]

B = 2 (the CFG pair), F = 17 latent frames, 32 x 32 patches, hidden 1152, 4096-wide captions (120 tokens).  Weights are random:
the timing does not depend on their values.  Prints the card and its power limit, then one JSON line; writes nothing unless
--out is given.
"""
import argparse
import json
import subprocess

import torch
import torch.nn.functional as F

B, FR, HP, WP, C, L, K = 2, 17, 32, 32, 1152, 120, 2
HBM_PEAK = 3.35e12


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def kernel_vs_eager(steps, warmup):
    from videosys_b200 import kernels as Kn

    dev, dt = "cuda", torch.bfloat16
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, FR, HP, WP, C, device=dev, generator=g).to(dt)
    w2 = (0.3 * torch.randn(C, 1, K, K, device=dev, generator=g)).to(dt)
    w1 = (0.3 * torch.randn(C, 1, K, device=dev, generator=g)).to(dt)
    b, lw, lb = [(0.3 * torch.randn(C, device=dev, generator=g)).to(dt) for _ in range(3)]
    t2, t1 = w2.reshape(C, -1).t().contiguous(), w1.reshape(C, -1).t().contiguous()
    pad = K - 1 if FR % 2 else 0
    S = HP * WP

    def spatial_ours():
        return Kn.kv_compress(x, t2, b, lw, lb, B, FR, HP, WP, (1, K, K), 0, 1e-5, round_conv=True)

    def spatial_eager():  # AttnProcessor2_0 :1184-1187 + :1197
        e = x.view(B * FR, S, C).permute(0, 2, 1).reshape(B * FR, C, HP, WP)
        e = F.conv2d(e, w2, b, stride=K, groups=C).reshape(B * FR, C, -1).permute(0, 2, 1)
        return F.layer_norm(e, (C,), lw, lb, 1e-5)

    def temporal_ours():
        return Kn.kv_compress(x, t1, b, lw, lb, B, FR, S, 1, (K, 1, 1), pad, 1e-5, round_conv=False)

    xt = x.view(B, FR, S, C).permute(0, 2, 1, 3).reshape(B * S, FR, C)  # the temporal block's [(b s), f, C]

    def temporal_eager():  # :1188-1193 + :1197
        e = xt.permute(0, 2, 1)
        e = torch.cat((e[:, :, :1].repeat(1, 1, pad), e), dim=2)
        return F.layer_norm(F.conv1d(e, w1, b, stride=K, groups=C).permute(0, 2, 1), (C,), lw, lb, 1e-5)

    res = {}
    for name, ours, eager in (("spatial", spatial_ours, spatial_eager), ("temporal", temporal_ours, temporal_eager)):
        nbytes = (x.numel() + ours().numel()) * 2
        ms_o, ms_e = _time(ours, steps * 20, warmup), _time(eager, steps * 20, warmup)
        res[name] = dict(ms=round(ms_o, 4), GBps=round(nbytes / ms_o / 1e6, 1),
                         share_of_hbm_peak=round(nbytes / ms_o / 1e-3 / HBM_PEAK, 3), eager_ms=round(ms_e, 4),
                         speedup_vs_eager=round(ms_e / ms_o, 2), bytes=nbytes)
    return res


def model_steps(steps, warmup, rounds):
    from videosys_b200.models.transformers.open_sora_plan_v110_transformer_3d import LatteT2V

    dev, dt = "cuda", torch.bfloat16
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, 4, FR, 2 * HP, 2 * WP, device=dev, generator=g).to(dt)
    enc = torch.randn(B, 1, L, 4096, device=dev, generator=g).to(dt)
    m = torch.ones(B, 1, L)
    t = torch.tensor([500, 500], device=dev)
    nets = {}
    for k in (1, 2):
        net = LatteT2V(num_layers=28, sample_size=(2 * HP, 2 * WP), video_length=FR, use_rope=False, compress_kv_factor=k)
        net = net.to(dt).to(dev).eval()
        with torch.no_grad():
            for p in net.parameters():
                p.copy_(0.02 * torch.randn(p.shape, device=dev, generator=g))
        nets[k] = net
    times = {1: [], 2: []}
    for _ in range(rounds):
        for k, net in nets.items():
            times[k].append(_time(lambda: net(x, timestep=t, encoder_hidden_states=enc, encoder_attention_mask=m,
                                              return_dict=False)[0], steps, warmup))
    return {f"compress_kv_factor_{k}": [round(v, 2) for v in ts] for k, ts in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    gpu = q[0] if q else torch.cuda.get_device_name()
    print(f"card, power limit, max SM clock: {gpu}", flush=True)
    res = dict(shape=dict(B=B, F=FR, patches=[HP, WP], hidden=C, text=L, k=K), gpu=gpu, kernel=kernel_vs_eager(a.steps, a.warmup),
               step_ms=model_steps(a.steps, a.warmup, a.rounds))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
