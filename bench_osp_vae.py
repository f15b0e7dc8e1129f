"""Open-Sora-Plan causal-VAE decode on one GPU: the native decoder (csrc/vae_conv.cu, csrc/vae_osp.cu) against the eager
torch / cuDNN chain of the same module (the stand-ins of tests/kernels_emul_osp_vae.py and tests/kernels_emul_vae.py, which
compute what the reference's eager decoder computes), in alternating rounds.

    python bench_osp_vae.py [--rounds 3]

Workloads, fp16, released widths (hidden_size 128, attention over 512 channels), random weights, each decoded tiled (the
pipeline's settings: 64-latent tiles, 8-frame chunks, overlap 0.25) and untiled:
  - v1.2.0, latents [1, 4, 8, 60, 80] -> 29 frames at 480 x 640;
  - v1.1.0 (TimeUpsampleRes2x, AttnBlock3D), latents [1, 4, 17, 64, 64] -> 65 frames at 512 x 512.
Prints the card and its power limit, then one JSON line.  The decoded frames of the two chains are compared at every size.
"""
import argparse
import json
import subprocess
import time

import torch

from oracle.gen_golden_osp_vae import V120_RELEASED, weights
from tests import kernels_emul as E
from tests import kernels_emul_osp_vae as EO
from tests import kernels_emul_vae as EV
from videosys_b200 import kernels
from videosys_b200.models.autoencoders import CausalVAEModelV110, CausalVAEModelV120

V110_RELEASED = dict(decoder_attention="AttnBlock3D", decoder_temporal_upsample=("", "", "TimeUpsampleRes2x", "TimeUpsampleRes2x"))
WORKLOADS = {"v120_29x480p": (CausalVAEModelV120, V120_RELEASED, (1, 4, 8, 60, 80)),
             "v110_65x512x512": (CausalVAEModelV110, V110_RELEASED, (1, 4, 17, 64, 64))}


def _time(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


class _Eager:
    """Patches the torch stand-ins over the kernels for the duration of a with-block."""

    PATCH = [(EV, EV.NAMES), (EO, EO.NAMES), (E, ["gemm_bias_act", "gemm_bias_residual"])]

    def __enter__(self):
        self.saved = {n: getattr(kernels, n) for _, names in self.PATCH for n in names}
        for mod, names in self.PATCH:
            for n in names:
                setattr(kernels, n, getattr(mod, n))

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(kernels, n, f)


def _tile(vae, tiled):
    vae.enable_tiling(tiled)
    vae.tile_overlap_factor, vae.tile_sample_min_size, vae.tile_latent_min_size = 0.25, 512, 64
    vae.tile_sample_min_size_t, vae.tile_latent_min_size_t = 29, 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_osp_vae.py needs a GPU"
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
    result = {"card": name, "power_limit": q}
    for wl, (cls, cfg, shape) in WORKLOADS.items():
        vae = cls(**cfg)
        vae.load_state_dict(weights(vae.state_dict(), "v120_released"))
        vae = vae.to(dt).cuda().eval()
        z = (0.18215 * torch.randn(*shape, generator=torch.Generator().manual_seed(0))).to(dt).cuda()
        for tiled in (True, False):
            _tile(vae, tiled)

            def eager():
                with _Eager():
                    return vae.decode(z)

            tn, te = [], []
            for r in range(args.rounds + 1):  # round 0 warms up: module loads, cuDNN algorithm choice
                t, ours = _time(lambda: vae.decode(z))
                u, ref = _time(eager)
                if r:
                    tn.append(t)
                    te.append(u)
            diff = (ours.float() - ref.float()).abs()
            key = f"{wl}_{'tiled' if tiled else 'untiled'}"
            result[key] = {"frames": list(ours.shape), "native_ms": round(min(tn), 1), "eager_ms": round(min(te), 1),
                           "native_ms_all": [round(t, 1) for t in tn], "eager_ms_all": [round(t, 1) for t in te],
                           "speedup": round(min(te) / min(tn), 3), "max_abs_diff": round(float(diff.max()), 4),
                           "mean_abs_diff": float(diff.mean()), "mean_abs": float(ref.float().abs().mean())}
            print(f"[{key}] {tuple(ours.shape)}: native {min(tn):.1f} ms, eager {min(te):.1f} ms per decode; "
                  f"|native - eager| max {float(diff.max()):.4f}, mean {float(diff.mean()):.2e}")
            del ours, ref
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
