"""OpenSora v1.2 VAE decode on one GPU: the native decoder (csrc/vae_conv.cu, csrc/vae_osp.cu) against the eager torch /
cuDNN chain of the same module (the stand-ins of tests/kernels_emul_opensora_vae.py, which compute what the reference's
eager decoder computes), in alternating rounds.

    python bench_opensora_vae.py [--rounds 2]

Workloads, bf16, released widths (temporal VAE and SDXL image decoder), random weights, the pipeline's micro-batching
(17-frame temporal chunks, 4 images per spatial pass):
  - 720p 9:16, 68 frames: latents [1, 4, 20, 90, 160];
  - 240p 9:16, 51 frames: latents [1, 4, 15, 30, 53].
Prints the card and its power limit, the FLOPs of the convolutions and GEMMs (counted from the shapes of the launches of
one native decode), then one JSON line.  The decoded frames of the two chains are compared.
"""
import argparse
import json
import subprocess
import time

import torch

from oracle.gen_golden_opensora_vae import weights
from tests import kernels_emul_opensora_vae as EOS
from videosys_b200 import kernels
from videosys_b200.models.autoencoders import VideoAutoencoderPipeline

WORKLOADS = {"720p_68f": ((1, 4, 20, 90, 160), 68), "240p_51f": ((1, 4, 15, 30, 53), 51)}


def _time(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


class _Eager:
    """Patches the torch stand-ins over the kernels for the duration of a with-block."""

    def __enter__(self):
        self.patch = EOS.stand_ins()
        self.saved = {n: getattr(kernels, n) for n in self.patch}
        for n, f in self.patch.items():
            setattr(kernels, n, f)

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(kernels, n, f)


def _flops(vae, z, nf):
    """(temporal, spatial) FLOPs of the convolutions and GEMMs of one native decode, from the launches' shapes."""
    kernels.PROFILE, kernels.PROFILE_KINDS = [], {"vae_conv3d", "gemm"}
    orig = vae.spatial_vae.decode
    marks = []

    def spatial(x):
        marks.append(len(kernels.PROFILE))
        return orig(x)

    vae.spatial_vae.decode = spatial
    try:
        vae.decode(z, num_frames=nf)
        torch.cuda.synchronize()
        works = [w for _, _, _, w in kernels.PROFILE]
    finally:
        kernels.PROFILE, kernels.PROFILE_KINDS = None, None
        del vae.spatial_vae.decode
    return sum(works[:marks[0]]), sum(works[marks[0]:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_opensora_vae.py needs a GPU"
    torch.backends.cudnn.benchmark = False
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        q = "unknown"
    print(f"card: {name}; power limit, max SM clock: {q}")
    torch.set_grad_enabled(False)
    vae = VideoAutoencoderPipeline()
    vae.load_state_dict(weights(vae.state_dict(), "released"))
    vae = vae.to(torch.bfloat16).cuda().eval()
    result = {"card": name, "power_limit": q}
    for wl, (shape, nf) in WORKLOADS.items():
        z = torch.randn(*shape, generator=torch.Generator().manual_seed(0)).to(torch.bfloat16).cuda()
        ft, fs = _flops(vae, z, nf)
        tn, te = [], []
        for r in range(args.rounds + 1):  # round 0 warms up: module loads, cuDNN algorithm choice
            t, ours = _time(lambda: vae.decode(z, num_frames=nf))
            with _Eager():
                u, ref = _time(lambda: vae.decode(z, num_frames=nf))
            if r:
                tn.append(t)
                te.append(u)
            if r < args.rounds:
                del ours, ref
                torch.cuda.empty_cache()
        diff = (ours.float() - ref.float()).abs()
        tflop = (ft + fs) / 1e12
        result[wl] = {"frames": list(ours.shape), "native_ms": round(min(tn), 1), "eager_ms": round(min(te), 1),
                      "native_ms_all": [round(t, 1) for t in tn], "eager_ms_all": [round(t, 1) for t in te],
                      "speedup": round(min(te) / min(tn), 3), "tflop_temporal": round(ft / 1e12, 2),
                      "tflop_spatial": round(fs / 1e12, 2), "native_tflops": round(tflop / (min(tn) / 1e3), 1),
                      "eager_tflops": round(tflop / (min(te) / 1e3), 1), "max_abs_diff": round(float(diff.max()), 4),
                      "mean_abs_diff": float(diff.mean()), "mean_abs": float(ref.float().abs().mean())}
        print(f"[{wl}] {tuple(ours.shape)}: {tflop:.1f} TFLOP (temporal {ft / 1e12:.1f}, spatial {fs / 1e12:.1f}); native "
              f"{min(tn):.1f} ms ({tflop / min(tn) * 1e3:.0f} TFLOP/s), eager {min(te):.1f} ms ({tflop / min(te) * 1e3:.0f} TFLOP/s); "
              f"|native - eager| max {float(diff.max()):.4f}, mean {float(diff.mean()):.2e}")
        del ours, ref, diff
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
