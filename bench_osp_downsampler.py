"""Measures Open-Sora-Plan v1.2.0's conv down-sampler path (downsampler="k333_s222") at the 29x480p shape on one GPU:

  - achieved HBM bandwidth of vsb_dwconv_shuffle and vsb_dwconv_ffn (bytes the algorithm must move: read the input once, write
    the output once) against the H100 SXM data-sheet 3.35 TB/s, next to the same pieces through the reference's eager ops
    (rearrange -> torch depth-wise conv + shortcut -> rearrange);
  - ms per full-depth (32-layer) transformer step with and without the down-sampler.

    python bench_osp_downsampler.py [--steps 10] [--warmup 3] [--out FILE.json]

B = 2 (the CFG pair), T = 8 latent frames, 30 x 40 patches, hidden 2304, 4096-wide captions (120 tokens).  Weights are random:
the timing does not depend on their values.  Prints one JSON line; writes nothing unless --out is given.
"""
import argparse
import json
import subprocess

import torch
import torch.nn.functional as F

B, T, HP, WP, C, L = 2, 8, 30, 40, 2304, 120
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


def kernels_vs_eager(steps, warmup):
    from videosys_b200 import kernels as K

    dev, dt = "cuda", torch.bfloat16
    g = torch.Generator(device=dev).manual_seed(0)
    N = T * HP * WP
    x = torch.randn(B, N, C, device=dev, generator=g).to(dt)
    w = (0.1 * torch.randn(C, 1, 3, 3, 3, device=dev, generator=g)).to(dt)
    b = (0.1 * torch.randn(C, device=dev, generator=g)).to(dt)
    taps = w.reshape(C, -1).t().contiguous()
    h = torch.randn(B * T, HP, WP, 2 * C, device=dev, generator=g).to(dt)
    convs = [((0.1 * torch.randn(2 * C, 1, k, k, device=dev, generator=g)).to(dt),
              (0.1 * torch.randn(2 * C, device=dev, generator=g)).to(dt)) for k in (5, 3, 1)]
    ftaps = torch.cat([cw.reshape(2 * C, -1).t() for cw, _ in convs], 0).contiguous()
    fbias = torch.stack([cb for _, cb in convs], 0).contiguous()

    def shuffle_ours():
        return K.dwconv_shuffle(x, taps, b, B, T, HP, WP, (3, 3, 3), (2, 2, 2))

    def shuffle_eager():  # DownSampler3d.forward: rearrange, Conv3d + shortcut, rearrange into the sub-grids
        xi = x.view(B, T, HP, WP, C).permute(0, 4, 1, 2, 3).contiguous()
        y = F.conv3d(xi, w, b, padding=1, groups=C) + xi
        y = y.view(B, C, T // 2, 2, HP // 2, 2, WP // 2, 2).permute(0, 3, 5, 7, 2, 4, 6, 1)
        return y.reshape(B * 8, -1, C)

    def ffn_ours():
        return K.dwconv_ffn(h, ftaps, fbias, B * T, HP, WP)

    def ffn_eager():  # FeedForward_Conv2d.forward between the GELU and project_out
        xi = h.permute(0, 3, 1, 2).contiguous()
        out = xi
        for (cw, cb), k in zip(convs, (5, 3, 1)):
            out = out + F.conv2d(xi, cw, cb, padding=k // 2, groups=2 * C)
        return out.permute(0, 2, 3, 1).reshape(B, N, 2 * C)

    res = {}
    for name, ours, eager, nbytes in (("dwconv_shuffle", shuffle_ours, shuffle_eager, 2 * x.numel() * 2),
                                      ("dwconv_ffn", ffn_ours, ffn_eager, 2 * h.numel() * 2)):
        ms_o, ms_e = _time(ours, steps * 10, warmup), _time(eager, steps * 10, warmup)
        res[name] = dict(ms=round(ms_o, 4), GBps=round(nbytes / ms_o / 1e6, 1), share_of_hbm_peak=round(nbytes / ms_o / 1e-3 / HBM_PEAK, 3),
                         eager_ms=round(ms_e, 4), speedup_vs_eager=round(ms_e / ms_o, 2), bytes=nbytes)
    return res


def model_step(downsampler, steps, warmup):
    from videosys_b200.models.transformers.open_sora_plan_v120_transformer_3d import OpenSoraT2V

    dev, dt = "cuda", torch.bfloat16
    net = OpenSoraT2V(num_attention_heads=24, attention_head_dim=96, num_layers=32, cross_attention_dim=2304, sample_size=(60, 80),
                      sample_size_t=T, caption_channels=4096, downsampler=downsampler).to(dt).to(dev).eval()
    g = torch.Generator(device=dev).manual_seed(1)
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(0.02 * torch.randn(p.shape, device=dev, generator=g))
    x = torch.randn(B, 4, T, 2 * HP, 2 * WP, device=dev, generator=g).to(dt)
    enc = torch.randn(B, 1, L, 4096, device=dev, generator=g).to(dt)
    m = torch.ones(B, 1, L)
    t = torch.tensor([500, 500], device=dev)

    def step():
        return net(x, timestep=t, encoder_hidden_states=enc, encoder_attention_mask=m, return_dict=False)[0]

    ms = _time(step, steps, warmup)
    del net
    torch.cuda.empty_cache()
    return round(ms, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = dict(shape=dict(B=B, T=T, patches=[HP, WP], hidden=C, text=L), gpu=q[0] if q else torch.cuda.get_device_name(),
               kernels=kernels_vs_eager(a.steps, a.warmup),
               step_ms=dict(downsampler_none=model_step(None, a.steps, a.warmup), k333_s222=model_step("k333_s222", a.steps, a.warmup)))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
