"""VAE decode on one GPU: the native decoders (csrc/vae_conv.cu, csrc/vae_osp.cu) against the eager torch / cuDNN chain
of the same modules (the stand-ins of tests/kernels_emul_vae.py, which compute what the reference's eager decoders
compute), in alternating rounds after a warm-up round.

    python bench_vae.py [--rounds 3] [cogvideox|osp|opensora|opensora_encode|latte|vchitect ...]    (all by default)

Workloads, random weights:
  - cogvideox: latents [1, 16, 13, 60, 90] (CogVideoX-2b, 49 frames at 480 x 720), fp16, released widths; decoded tiled
    (the pipeline default) and untiled; then the per-kernel rates of the CogVideoX kernels.
  - osp: fp16, released widths (hidden_size 128, attention over 512 channels), each decoded tiled (the pipeline's
    settings: 64-latent tiles, 8-frame chunks, overlap 0.25) and untiled:
      v1.2.0, latents [1, 4, 8, 60, 80] -> 29 frames at 480 x 640;
      v1.1.0 (TimeUpsampleRes2x, AttnBlock3D), latents [1, 4, 17, 64, 64] -> 65 frames at 512 x 512.
  - opensora: bf16, released widths (temporal VAE and SDXL image decoder), the pipeline's micro-batching (17-frame
    temporal chunks, 4 images per spatial pass), with the FLOPs of the convolutions and GEMMs counted from the shapes of
    the launches of one native decode:
      720p 9:16, 68 frames: latents [1, 4, 20, 90, 160];
      240p 9:16, 51 frames: latents [1, 4, 15, 30, 53].
  - opensora_encode: bf16, released widths, OpenSoraVAEEncoder.encode with the pipeline's micro-batching (4 images per
    spatial pass, 17-frame temporal chunks), the posterior noise drawn under one seed in both chains:
      one 720p 9:16 image (an image-to-video reference): video [1, 3, 1, 720, 1280];
      a 51-frame 720p clip (a looped generation's re-encode): video [1, 3, 51, 720, 1280];
      a 51-frame 240p clip: video [1, 3, 51, 240, 426];
    then the rates of the strided convolution on its own (Downsample2D at the first level, the temporal stride-2 conv).
  - latte: fp16, released widths, latents [1, 4, 16, 64, 64] (16 frames at 512 x 512) as LattePipeline decodes them:
    the SVD temporal decoder on chunks of 14 + 2 frames, and the image VAE (enable_vae_temporal_decoder=False); then the
    rates of the time-axis convolution at the temporal decoder's top level (128 channels, 512 x 512, 14 frames): plain,
    with the residual + AlphaBlender epilogue, and the same result unfused (residual epilogue, then a vae_mix pass).
  - vchitect: bf16, released widths, 16 latent channels, latents [1, 40, 16, 36, 60] (40 frames at 288 x 480), decoded as
    VchitectXLPipeline does (several frames per pass).
For OpenSora (decode and encode), Latte and Vchitect the FLOPs of the convolutions and GEMMs are counted from the shapes of the launches of
one native decode.  Prints the card and its power limit, then one JSON line per model.  For Open-Sora-Plan, OpenSora,
Latte and Vchitect the decoded frames of the two chains are compared.
"""
import argparse
import contextlib
import json
import subprocess
import time

import torch

from oracle import gen_golden_cogvideox_vae as GC, gen_golden_opensora_vae as GS, gen_golden_osp_vae as GP
from oracle import gen_golden_latte_vae as GL
from tests import kernels_emul_vae_down as ED
from tests import kernels_emul_vae_time as EV
from videosys_b200 import kernels
from videosys_b200.models.autoencoders import (AutoencoderKL, AutoencoderKLCogVideoX, AutoencoderKLTemporalDecoder,
                                               CausalVAEModelV110, CausalVAEModelV120, OpenSoraVAEEncoder,
                                               VideoAutoencoderPipeline)
from videosys_b200.pipelines._common import decode_image_frames


# ---- the shared harness ----
def _time(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


@contextlib.contextmanager
def _eager():
    """The torch stand-ins patched over the kernels for the duration of a with-block."""
    patch = {**EV.stand_ins(), **ED.stand_ins()}
    saved = {n: getattr(kernels, n) for n in patch}
    for n, f in patch.items():
        setattr(kernels, n, f)
    try:
        yield
    finally:
        for n, f in saved.items():
            setattr(kernels, n, f)


def _rounds(decode, rounds):
    """Round 0 warms up (module loads, cuDNN algorithm choice); rounds 1.. time the native, then the eager decode.
    Returns the timings and the last round's two outputs."""
    tn, te = [], []
    for r in range(rounds + 1):
        ours = ref = None  # the previous round's outputs are freed before the next decode
        t, ours = _time(decode)
        with _eager():
            u, ref = _time(decode)
        if r:
            tn.append(t)
            te.append(u)
    return tn, te, ours, ref


def _times(tn, te):
    return {"native_ms": round(min(tn), 1), "eager_ms": round(min(te), 1), "native_ms_all": [round(t, 1) for t in tn],
            "eager_ms_all": [round(t, 1) for t in te], "speedup": round(min(te) / min(tn), 3)}


def _diff(ours, ref):
    diff = (ours.float() - ref.float()).abs()
    return {"max_abs_diff": round(float(diff.max()), 4), "mean_abs_diff": float(diff.mean()),
            "mean_abs": float(ref.float().abs().mean())}


def _events(fn, reps):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


# ---- CogVideoX ----
def kernel_rates(dt):
    """ms, TFLOP/s (conv) or GB/s (norm, upsample) of each CogVideoX kernel at decoder shapes."""
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


def cogvideox(rounds):
    dt = torch.float16
    vae = AutoencoderKLCogVideoX(**GC.CASES["released_f3"][0])
    vae.load_state_dict(GC.weights(vae.state_dict(), "released_f3"))
    vae = vae.to(dt).cuda().eval()
    z = torch.randn(1, 16, 13, 60, 90, generator=torch.Generator().manual_seed(0)).to(dt).cuda()
    result = {"workload": "cogvideox_vae_decode_1x16x13x60x90_fp16"}
    for tiled in (True, False):
        vae.enable_tiling() if tiled else vae.disable_tiling()
        tn, te, _, _ = _rounds(lambda: vae.decode(z), rounds)
        key = "tiled" if tiled else "untiled"
        result[key] = _times(tn, te)
        print(f"[cogvideox {key}] native {min(tn):.1f} ms, eager {min(te):.1f} ms per decode")
    result["kernels"] = kernel_rates(dt)
    return result


# ---- Open-Sora-Plan ----
OSP_V110_RELEASED = dict(decoder_attention="AttnBlock3D", decoder_temporal_upsample=("", "", "TimeUpsampleRes2x", "TimeUpsampleRes2x"))
OSP_WORKLOADS = {"v120_29x480p": (CausalVAEModelV120, GP.V120_RELEASED, (1, 4, 8, 60, 80)),
                 "v110_65x512x512": (CausalVAEModelV110, OSP_V110_RELEASED, (1, 4, 17, 64, 64))}


def _osp_tile(vae, tiled):
    vae.enable_tiling(tiled)
    vae.tile_overlap_factor, vae.tile_sample_min_size, vae.tile_latent_min_size = 0.25, 512, 64
    vae.tile_sample_min_size_t, vae.tile_latent_min_size_t = 29, 8


def osp(rounds):
    result = {}
    for wl, (cls, cfg, shape) in OSP_WORKLOADS.items():
        vae = cls(**cfg)
        vae.load_state_dict(GP.weights(vae.state_dict(), "v120_released"))
        vae = vae.to(torch.float16).cuda().eval()
        z = (0.18215 * torch.randn(*shape, generator=torch.Generator().manual_seed(0))).to(torch.float16).cuda()
        for tiled in (True, False):
            _osp_tile(vae, tiled)
            tn, te, ours, ref = _rounds(lambda: vae.decode(z), rounds)
            key = f"{wl}_{'tiled' if tiled else 'untiled'}"
            result[key] = {"frames": list(ours.shape), **_times(tn, te), **_diff(ours, ref)}
            print(f"[osp {key}] {tuple(ours.shape)}: native {min(tn):.1f} ms, eager {min(te):.1f} ms per decode; "
                  f"|native - eager| max {result[key]['max_abs_diff']:.4f}, mean {result[key]['mean_abs_diff']:.2e}")
            del ours, ref
            torch.cuda.empty_cache()
    return result


# ---- OpenSora v1.2 ----
OPENSORA_WORKLOADS = {"720p_68f": ((1, 4, 20, 90, 160), 68), "240p_51f": ((1, 4, 15, 30, 53), 51)}


def _opensora_flops(vae, z, nf):
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


def opensora(rounds):
    vae = VideoAutoencoderPipeline()
    vae.load_state_dict(GS.weights(vae.state_dict(), "released"))
    vae = vae.to(torch.bfloat16).cuda().eval()
    result = {}
    for wl, (shape, nf) in OPENSORA_WORKLOADS.items():
        z = torch.randn(*shape, generator=torch.Generator().manual_seed(0)).to(torch.bfloat16).cuda()
        ft, fs = _opensora_flops(vae, z, nf)
        tn, te, ours, ref = _rounds(lambda: vae.decode(z, num_frames=nf), rounds)
        tflop = (ft + fs) / 1e12
        result[wl] = {"frames": list(ours.shape), **_times(tn, te), "tflop_temporal": round(ft / 1e12, 2),
                      "tflop_spatial": round(fs / 1e12, 2), "native_tflops": round(tflop / (min(tn) / 1e3), 1),
                      "eager_tflops": round(tflop / (min(te) / 1e3), 1), **_diff(ours, ref)}
        print(f"[opensora {wl}] {tuple(ours.shape)}: {tflop:.1f} TFLOP (temporal {ft / 1e12:.1f}, spatial {fs / 1e12:.1f}); "
              f"native {min(tn):.1f} ms ({tflop / min(tn) * 1e3:.0f} TFLOP/s), eager {min(te):.1f} ms "
              f"({tflop / min(te) * 1e3:.0f} TFLOP/s); |native - eager| max {result[wl]['max_abs_diff']:.4f}, "
              f"mean {result[wl]['mean_abs_diff']:.2e}")
        del ours, ref
        torch.cuda.empty_cache()
    return result


# ---- Latte and Vchitect-2.0 ----
def _flops(decode):
    """FLOPs of the convolutions and GEMMs of one native decode (or encode), from the launches' shapes."""
    kernels.PROFILE, kernels.PROFILE_KINDS = [], {"vae_conv3d", "vae_conv_time", "vae_conv_down", "gemm"}
    try:
        decode()
        torch.cuda.synchronize()
        return sum(w for _, _, _, w in kernels.PROFILE)
    finally:
        kernels.PROFILE, kernels.PROFILE_KINDS = None, None


def _run(tag, decode, rounds):
    flop = _flops(decode)
    tn, te, ours, ref = _rounds(decode, rounds)
    res = {"frames": list(ours.shape), **_times(tn, te), "tflop": round(flop / 1e12, 2),
           "native_tflops": round(flop / 1e12 / (min(tn) / 1e3), 1), "eager_tflops": round(flop / 1e12 / (min(te) / 1e3), 1),
           **_diff(ours, ref)}
    print(f"[{tag}] {tuple(ours.shape)}: {flop / 1e12:.2f} TFLOP; native {min(tn):.1f} ms ({res['native_tflops']} TFLOP/s), "
          f"eager {min(te):.1f} ms ({res['eager_tflops']} TFLOP/s); |native - eager| max {res['max_abs_diff']:.4f}, "
          f"mean {res['mean_abs_diff']:.2e} (on the [-1, 1] scale)")
    return res


def conv_time_rates(dt):
    """ms and TFLOP/s of vae_conv_time at the temporal decoder's top level, with and without the mix epilogue."""
    g = torch.Generator(device="cuda").manual_seed(0)
    T, H, W, C = 14, 512, 512, 128
    x = torch.randn(1, T + 2, H, W, C, device="cuda", generator=g).to(dt)
    xs = torch.randn(1, T, H, W, C, device="cuda", generator=g).to(dt)
    wp = kernels.pack_conv_weight((0.05 * torch.randn(C, C, 3, 1, 1, device="cuda", generator=g)).to(dt))
    b = torch.zeros(C, device="cuda", dtype=dt)
    flop = 2 * T * H * W * C * C * 3
    res = {}
    for name, kw in (("conv_time_128_512x512_t14", {}), ("conv_time_mix_128_512x512_t14", dict(resid=xs, mix=(0.25, 0.75)))):
        ms = _events(lambda: kernels.vae_conv_time(x, wp, b, C, 3, **kw), 10)
        res[name] = {"ms": round(ms, 3), "tflops": round(flop / ms / 1e9, 1)}
    # the same result unfused: the residual in the conv epilogue, then the AlphaBlender as a separate vae_mix pass
    ms = _events(lambda: kernels.vae_mix(xs, kernels.vae_conv_time(x, wp, b, C, 3, resid=xs), 0.25, 0.75), 10)
    res["conv_time_resid_then_vae_mix_128_512x512_t14"] = {"ms": round(ms, 3), "tflops": round(flop / ms / 1e9, 1)}
    return res


def latte(rounds):
    dt = torch.float16
    z = (torch.randn(1, 4, 16, 64, 64, generator=torch.Generator().manual_seed(0)) / 0.18215).to(dt).cuda()
    frames = z.permute(0, 2, 1, 3, 4).reshape(16, 4, 64, 64)  # the pipeline's (b f) c h w, already scaled
    result = {"workload": "latte_vae_decode_1x4x16x64x64_fp16"}
    for key, cls in (("temporal_decoder", AutoencoderKLTemporalDecoder), ("sd_vae", AutoencoderKL)):
        vae = cls()
        vae.load_state_dict(GS.weights(vae.state_dict(), "released"))
        vae = vae.to(dt).cuda().eval()
        if cls is AutoencoderKLTemporalDecoder:  # LattePipeline.decode_video: chunks of 14 frames
            decode = lambda: torch.cat([vae.decode(frames[i:i + 14], num_frames=len(frames[i:i + 14])).sample  # noqa: E731
                                        for i in range(0, 16, 14)])
        else:
            decode = lambda: decode_image_frames(vae, frames)  # noqa: E731
        result[key] = _run(f"latte {key}", decode, rounds)
        del vae
        torch.cuda.empty_cache()
    result["kernels"] = conv_time_rates(dt)
    return result


def vchitect(rounds):
    dt = torch.bfloat16
    vae = AutoencoderKL(latent_channels=16, use_post_quant_conv=False)
    vae.load_state_dict(GS.weights(vae.state_dict(), "released"))
    vae = vae.to(dt).cuda().eval()
    z = torch.randn(1, 40, 16, 36, 60, generator=torch.Generator().manual_seed(0)).to(dt).cuda()
    z = (z / GL.VCH_SCALE) + GL.VCH_SHIFT
    return {"workload": "vchitect_vae_decode_1x40x16x36x60_bf16", **_run("vchitect", lambda: decode_image_frames(vae, z[0]), rounds)}


# ---- OpenSora v1.2 encoder ----
OPENSORA_ENCODE_WORKLOADS = {"720p_image": (1, 3, 1, 720, 1280), "720p_51f": (1, 3, 51, 720, 1280),
                             "240p_51f": (1, 3, 51, 240, 426)}


def conv_down_rates(dt):
    """ms and TFLOP/s of vae_conv_down at the encoders' shapes."""
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {}
    for name, (N, T, H, W, C, kt) in {"down2d_128_720x1280_n4": (4, 1, 720, 1280, 128, 1),
                                      "down2d_512_180x320_n4": (4, 1, 180, 320, 512, 1),
                                      "down_t_256_90x160_t20": (1, 20, 90, 160, 256, 3)}.items():
        x = torch.randn(N, T, H, W, C, device="cuda", generator=g).to(dt)
        wp = kernels.pack_conv_weight((0.02 * torch.randn(C, C, kt, 3, 3, device="cuda", generator=g)).to(dt))
        b = torch.zeros(C, device="cuda", dtype=dt)
        out = kernels.vae_conv_down(x, wp, b, C, kt)
        flop = 2 * out.numel() * C * kt * 9
        ms = _events(lambda: kernels.vae_conv_down(x, wp, b, C, kt), 10)
        res[name] = {"ms": round(ms, 3), "tflops": round(flop / ms / 1e9, 1)}
    return res


def opensora_encode(rounds):
    dt = torch.bfloat16
    enc = OpenSoraVAEEncoder()
    enc.load_state_dict(GS.weights(enc.state_dict(), "released"))
    enc = enc.to(dt).cuda().eval()

    def encode(x):
        torch.manual_seed(0)  # the same posterior noise in both chains
        return enc.encode(x)

    result = {}
    for wl, shape in OPENSORA_ENCODE_WORKLOADS.items():
        x = (2 * torch.rand(*shape, generator=torch.Generator().manual_seed(0)) - 1).to(dt).cuda()
        result[wl] = _run(f"opensora_encode {wl}", lambda: encode(x), rounds)
        del x
        torch.cuda.empty_cache()
    result["kernels"] = conv_down_rates(dt)
    return result


MODELS = {"cogvideox": cogvideox, "osp": osp, "opensora": opensora, "opensora_encode": opensora_encode, "latte": latte,
          "vchitect": vchitect}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("models", nargs="*", metavar="MODEL", help=f"any of {', '.join(MODELS)} (default: all)")
    args = ap.parse_args()
    unknown = [m for m in args.models if m not in MODELS]
    if unknown:
        ap.error(f"unknown model(s) {unknown}: choose from {list(MODELS)}")
    assert torch.cuda.is_available(), "bench_vae.py needs a GPU"
    torch.backends.cudnn.benchmark = False
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        q = "unknown"
    print(f"card: {name}; power limit, max SM clock: {q}")
    torch.set_grad_enabled(False)
    for m in args.models or list(MODELS):
        print(json.dumps({"model": m, "card": name, "power_limit": q, **MODELS[m](args.rounds)}))
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
