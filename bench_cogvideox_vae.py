"""CogVideoX VAE decode on one GPU: the native decoder (csrc/vae_conv.cu) against the eager torch / cuDNN chain of the same
module (the stand-ins of tests/kernels_emul_vae.py, which compute what the reference's eager decoder computes), in
alternating rounds, plus the per-kernel rates of the new kernels.

    python bench_cogvideox_vae.py [--rounds 3]

Workload: latents [1, 16, 13, 60, 90] (CogVideoX-2b, 49 frames at 480 x 720), fp16, released widths, random weights; decoded
tiled (the pipeline default) and untiled.  Prints the card and its power limit, then one JSON line.
"""
import argparse
import json
import subprocess
import time

import torch
import torch.nn.functional as F

from oracle.gen_golden_cogvideox_vae import CASES, weights
from tests import kernels_emul_vae as EV
from videosys_b200 import kernels
from videosys_b200.models.autoencoders import AutoencoderKLCogVideoX


def _time(fn, reps=1):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def _events(fn, reps):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


class _Eager:
    """Patches the torch stand-ins over the kernels for the duration of a with-block."""

    def __enter__(self):
        self.saved = {n: getattr(kernels, n) for n in EV.NAMES + ["gemm_bias_act"]}
        for n in EV.NAMES:
            setattr(kernels, n, getattr(EV, n))
        kernels.gemm_bias_act = lambda a, w, bias=None, act=0, out=None: F.linear(a, w, bias)

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(kernels, n, f)


def kernel_rates(dt):
    """ms, TFLOP/s (conv) or GB/s (norm, upsample) of each new kernel at decoder shapes."""
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g).to(dt)  # noqa: E731
    res = {}
    for name, (T, H, W, cin, cout, kt) in {"conv_512_60x90": (3, 60, 90, 512, 512, 3), "conv_128_240x360": (9, 240, 360, 128, 128, 3),
                                           "conv_upsample_256_240x360": (9, 240, 360, 256, 256, 1),
                                           "conv_out_128to3_240x360": (9, 240, 360, 128, 3, 3)}.items():
        x = rnd(1, T + kt - 1, H, W, cin)
        wp = kernels.pack_conv_weight(rnd(cout, cin, kt, 3, 3) * 0.02)
        b = rnd(cout)
        ms = _events(lambda: kernels.vae_conv3d(x, wp, b, cout, kt), 10)
        res[name] = {"ms": round(ms, 4), "tflops": round(2 * T * H * W * cout * cin * kt * 9 / ms / 1e9, 1)}
    f = rnd(1, 9, 240, 360, 128)
    ms = _events(lambda: kernels.vae_groupnorm_stats(f, 32, 1e-6), 20)
    res["groupnorm_stats_128_240x360_t9"] = {"ms": round(ms, 4), "gbs": round(f.numel() * 2 / ms / 1e6, 1)}
    stats = kernels.vae_groupnorm_stats(f, 32, 1e-6)
    zyb, out = rnd(1, 3, 30, 45, 256), torch.empty(1, 11, 240, 360, 128, device="cuda", dtype=dt)
    gam, bet = rnd(128), rnd(128)
    ms = _events(lambda: kernels.vae_spatial_norm_silu(f, stats, gam, bet, zyb, out, 2), 20)
    res["spatial_norm_silu_128_240x360_t9"] = {"ms": round(ms, 4), "gbs": round(2 * f.numel() * 2 / ms / 1e6, 1)}
    u = rnd(1, 5, 120, 180, 256)
    ms = _events(lambda: kernels.vae_upsample2x(u, True), 20)
    res["upsample2x_256_120x180_t5"] = {"ms": round(ms, 4), "gbs": round((u.numel() + 4 * 9 * 120 * 180 * 256) * 2 / ms / 1e6, 1)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_cogvideox_vae.py needs a GPU"
    torch.backends.cudnn.benchmark = False
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        q = "unknown"
    print(f"card: {name}; power limit, max SM clock: {q}")
    dt = torch.float16
    torch.set_grad_enabled(False)
    vae = AutoencoderKLCogVideoX(**CASES["released_f3"][0])
    vae.load_state_dict(weights(vae.state_dict(), "released_f3"))
    vae = vae.to(dt).cuda().eval()
    z = torch.randn(1, 16, 13, 60, 90, generator=torch.Generator().manual_seed(0)).to(dt).cuda()
    result = {"workload": "cogvideox_vae_decode_1x16x13x60x90_fp16", "card": name, "power_limit": q}
    for tiled in (True, False):
        vae.enable_tiling() if tiled else vae.disable_tiling()
        native = lambda: vae.decode(z)  # noqa: E731

        def eager():
            with _Eager():
                return vae.decode(z)

        native(), eager()  # warm-up: module loads, cuDNN algorithm choice
        tn, te = [], []
        for _ in range(args.rounds):
            tn.append(_time(native))
            te.append(_time(eager))
        key = "tiled" if tiled else "untiled"
        result[key] = {"native_ms": round(min(tn), 1), "eager_ms": round(min(te), 1), "native_ms_all": [round(t, 1) for t in tn],
                       "eager_ms_all": [round(t, 1) for t in te], "speedup": round(min(te) / min(tn), 3)}
        print(f"[{key}] native {min(tn):.1f} ms, eager {min(te):.1f} ms per decode")
    result["kernels"] = kernel_rates(dt)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
