"""Times ``kernels.gemm_bias_act`` / ``kernels.gemm_bias_residual`` alone at the shapes the model front ends hand them:

  qkv          OpenSora v1.2 720p attn.qkv: M = 2 x 20 x 3600 tokens, N 3456, K 1152, + bias
  attn_proj    attn.proj: N 1152, K 1152, + bias, gate (modulation row 2), per-frame t / t0 select, residual, in place
  q_linear     cross_attn.q_linear: N 1152, K 1152, + bias
  cross_proj   cross_attn.proj: N 1152, K 1152, + bias, residual, in place
  fc1          mlp.fc1: N 4608, K 1152, + bias, tanh-GELU
  fc2          mlp.fc2: N 1152, K 4608, + bias, gate (row 5), frame select, residual, in place
  k2304        N 1152, K 2304, + bias: with q_linear (K 1152) and k4608 the time against K, whose intercept is the
  k4608        fixed cost of a tile (pipeline fill, epilogue, store) that the mainloop does not hide
  cogvideox    CogVideoX-2B fp16 Linear: M = 2 x 17 776, N 1920, K 1920, + bias
  cogvideox_ff its feed-forward in: N 7680, K 1920, + bias, tanh-GELU
  osp_ff       Open-Sora-Plan v1.2.0 480p feed-forward in: M = 2 x 9600, N 9216, K 2304, + bias, tanh-GELU
  osp_erf      its conv feed-forward in: N 4608, K 2304, + bias, erf-GELU
  gelu_k1536   tanh-GELU at K 1536 and 3072 (M 36 000, N 4608): with fc1 (K 1152) and the two above, where the GELU
  gelu_k3072   epilogue stops paying for a kernel of its own
  t_block      the t_block Linear: M = 2 (a CFG pair), N 6912, K 1152
  m4096_*      M 4096 and N 4608 (m4096_*) or N 1024 (n1024_*): too few tiles for the 256 x 128 kernel, so these time
  n1024_*      the instances no shape above reaches: the ping-pong kernel's tanh- / erf-GELU epilogues (K 1152), the
               one-tile-per-CTA kernel's GELU epilogues (K 2304) at tile widths 192 and 128, and its 128-wide bias-only
               tile (n1024, K 1152)

FP8 twins (``<name>_fp8``) of the six OpenSora 720p Linears run ``kernels.gemm_fp8_bias_act`` / ``_residual`` on e4m3
operands with the same epilogue; where the FP8 mode of the model quantizes the input in a pass of its own (attn_proj,
q_linear, cross_proj, fc2) that pass (``kernels.quant_rows_fp8``) is inside the timed launch, so their rate is FLOPs
over quantization + GEMM.  qkv and fc1 take their codes from the modulate kernel.  ``quant_k1152`` / ``quant_k4608``
time the quantization alone at M = 2 x 20 x 3600, as bytes (2 B read + 1 B written per element, 4 B per row) against
3.35 TB/s.

    python bench_gemm.py [--iters 20] [--warmup 3] [--rounds 3] [--shapes a,b] [--no-cublas] [--out FILE.json]

Inputs are seeded, so two builds given the same arguments can be compared output for output: every shape prints the
kernel instance the library dispatches it to and the SHA-256 of the output of one launch on fresh inputs.  Rates are
2 M N K FLOPs over the kernel time from CUDA events around --iters back-to-back launches; the median over --rounds is
reported.  As a ceiling for comparison the same operands also go through torch.nn.functional.linear (cuBLAS, bias only:
no gate or residual); the library never calls cuBLAS.  The card's name, power limit and SM clock (sampled while the
launches run) are part of the result.  Needs a CUDA device.  Writes nothing unless --out is given.
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

M720 = 2 * 20 * 3600
# name: (M, N, K, dtype, epilogue); epilogue: act 0 / 1 / 2 (none, tanh-GELU, erf-GELU) of gemm_bias_act, or
# ("res", gate_row) of gemm_bias_residual
SHAPES = {
    "qkv": (M720, 3456, 1152, torch.bfloat16, 0),
    "attn_proj": (M720, 1152, 1152, torch.bfloat16, ("res", 2)),
    "q_linear": (M720, 1152, 1152, torch.bfloat16, 0),
    "cross_proj": (M720, 1152, 1152, torch.bfloat16, ("res", -1)),
    "fc1": (M720, 4608, 1152, torch.bfloat16, 1),
    "fc2": (M720, 1152, 4608, torch.bfloat16, ("res", 5)),
    "k2304": (M720, 1152, 2304, torch.bfloat16, 0),
    "k4608": (M720, 1152, 4608, torch.bfloat16, 0),
    "cogvideox": (2 * 17776, 1920, 1920, torch.float16, 0),
    "cogvideox_ff": (2 * 17776, 7680, 1920, torch.float16, 1),
    "osp_ff": (2 * 9600, 9216, 2304, torch.bfloat16, 1),
    "osp_erf": (2 * 9600, 4608, 2304, torch.bfloat16, 2),
    "gelu_k1536": (36000, 4608, 1536, torch.bfloat16, 1),
    "gelu_k3072": (36000, 4608, 3072, torch.bfloat16, 1),
    "t_block": (2, 6912, 1152, torch.bfloat16, 0),
    "m4096_tanh": (4096, 4608, 1152, torch.bfloat16, 1),
    "m4096_erf": (4096, 4608, 1152, torch.bfloat16, 2),
    "m4096_tanh_k2304": (4096, 4608, 2304, torch.bfloat16, 1),
    "m4096_erf_k2304": (4096, 4608, 2304, torch.bfloat16, 2),
    "n1024": (4096, 1024, 1152, torch.bfloat16, 0),
    "n1024_tanh": (4096, 1024, 2304, torch.bfloat16, 1),
    "n1024_erf": (4096, 1024, 2304, torch.bfloat16, 2),
}
# name: (the bf16 shape, whether the timed launch includes the activation's quantization)
FP8_SHAPES = {"qkv_fp8": ("qkv", False), "attn_proj_fp8": ("attn_proj", True), "q_linear_fp8": ("q_linear", True),
              "cross_proj_fp8": ("cross_proj", True), "fc1_fp8": ("fc1", False), "fc2_fp8": ("fc2", True)}
QUANT_SHAPES = {"quant_k1152": (M720, 1152), "quant_k4608": (M720, 4608)}
HBM_BYTES_PER_S = 3.35e12
for _n, (_b, _) in FP8_SHAPES.items():
    SHAPES[_n] = SHAPES[_b]
for _n, (_m, _k) in QUANT_SHAPES.items():
    SHAPES[_n] = (_m, _k, _k, torch.bfloat16, "quant")
B720, T720, S720 = 2, 20, 3600


def make_call(name, dev, seed):
    """Seeded inputs of one shape; returns (launch(), reset(), output tensor, cuBLAS launch(), FLOPs per launch)."""
    from videosys_b200 import kernels

    M, N, K, dt, epi = SHAPES[name]
    g = torch.Generator(device=dev).manual_seed(seed)

    def rnd(*shape, std=1.0):
        return (std * torch.randn(*shape, device=dev, generator=g)).to(dt)

    a, w, bias = rnd(M, K), rnd(N, K, std=K**-0.5), rnd(N, std=0.1)
    def cublas():
        torch.nn.functional.linear(a, w, bias)

    if epi == "quant":
        res = []

        def launch():
            res[:] = kernels.quant_rows_fp8(a)
        launch()
        return launch, (lambda: None), lambda: res[0], cublas, 3 * M * K + 4 * M
    fp8 = name in FP8_SHAPES
    if fp8:
        wq, ws = kernels.quant_rows_fp8(w)
        aq = kernels.quant_rows_fp8(a)
        with_quant = FP8_SHAPES[name][1]

        def gemm_a():
            return kernels.quant_rows_fp8(a) if with_quant else aq

    if isinstance(epi, tuple):
        gate_row = epi[1]
        x0 = rnd(M, N)
        x = x0.clone()
        mod = rnd(2, B720, 6, N, std=0.5) if gate_row >= 0 else None
        mask = torch.ones(B720, T720, device=dev, dtype=torch.uint8)
        mask[0, 3] = 0
        mask[1, 17] = 0

        def launch():
            if fp8:
                kernels.gemm_fp8_bias_residual(*gemm_a(), wq, ws, bias, x, *((mod, mask, gate_row, B720, T720, S720)
                                                                              if gate_row >= 0 else ()))
            elif gate_row >= 0:
                kernels.gemm_bias_residual(a, w, bias, x, mod, mask, gate_row, B720, T720, S720)
            else:
                kernels.gemm_bias_residual(a, w, bias, x)

        def reset():
            x.copy_(x0)
        return launch, reset, x, cublas, 2 * M * N * K
    out = torch.empty(M, N, device=dev, dtype=dt)

    def launch():
        if fp8:
            kernels.gemm_fp8_bias_act(*gemm_a(), wq, ws, bias, act=epi, out=out)
        else:
            kernels.gemm_bias_act(a, w, bias, act=epi, out=out)
    return launch, (lambda: None), out, cublas, 2 * M * N * K


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def _time(fn, iters, warmup):
    from bench import ClockSampler

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    return e0.elapsed_time(e1) / iters, clocks["sm_mhz"]


def kernel_of(name):
    """The kernel instance the library launches for a shape."""
    from videosys_b200 import kernels

    M, N, K, _, epi = SHAPES[name]
    if epi == "quant":
        return "quant_rows_fp8_kernel"
    if name in FP8_SHAPES:
        q = "quant_rows_fp8_kernel + " if FP8_SHAPES[name][1] else ""
        return q + kernels.gemm_fp8_kernel_name(M, N, K, act=0 if isinstance(epi, tuple) else epi, residual=isinstance(epi, tuple))
    if isinstance(epi, tuple):
        return kernels.gemm_kernel_name(M, N, K, residual=True)
    return kernels.gemm_kernel_name(M, N, K, act=epi)


def run_shape(name, seed, iters, warmup, cublas):
    if not torch.cuda.is_available():
        raise SystemExit(f"bench_gemm.py: {name} needs a CUDA device")
    launch, reset, out, ref, flops = make_call(name, "cuda", seed)
    reset()
    launch()
    torch.cuda.synchronize()
    quant = SHAPES[name][4] == "quant"
    digest = hashlib.sha256((out()[0].view(torch.uint8) if quant else out.view(torch.int16)).cpu().numpy().tobytes()).hexdigest()
    ms, mhz = _time(launch, iters, warmup)
    res = dict(ms=round(ms, 4), tflops=round(flops / (ms * 1e-3) / 1e12, 1), sha256=digest, sm_mhz=mhz)
    if quant:  # bytes, not FLOPs: the rate is TB/s, and its share of the HBM bandwidth
        res.update(tflops=None, tb_s=round(flops / (ms * 1e-3) / 1e12, 3), hbm_share=round(flops / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
        cublas = False
    if name in FP8_SHAPES:
        cublas = False
    if cublas:
        ms_ref, _ = _time(ref, iters, warmup)
        res["cublas_ms"] = round(ms_ref, 4)
        res["cublas_tflops"] = round(flops / (ms_ref * 1e-3) / 1e12, 1)
    del launch, reset, out, ref
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="time every shape this many times (in turn); the median is reported")
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated subset of " + ", ".join(SHAPES))
    ap.add_argument("--no-cublas", action="store_true", help="skip the torch.nn.functional.linear ceiling")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    names = [s for s in a.shapes.split(",") if s]
    bad = [s for s in names if s not in SHAPES]
    if bad:
        ap.error(f"unknown shapes {bad}")
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm.py needs a CUDA device")
    runs = {}
    for r in range(a.rounds):
        for i, name in enumerate(names):
            m = run_shape(name, a.seed + i, a.iters, a.warmup, not a.no_cublas and r == 0)
            cb = f"  cublas {m['cublas_tflops']:6.1f} TFLOP/s" if "cublas_ms" in m else ""
            rate = f"{m['tb_s']:6.3f} TB/s ({100 * m['hbm_share']:.0f} % of HBM)" if "tb_s" in m else f"{m['tflops']:6.1f} TFLOP/s"
            print(f"round {r} {name:11s} {kernel_of(name):25s} {m['ms']:9.4f} ms {rate}{cb}  "
                  f"sm {m['sm_mhz']} MHz  sha256 {m['sha256']}", flush=True)
            runs.setdefault(name, []).append(m)
    res = dict(gpu=gpu_info(), iters=a.iters, rounds=a.rounds, shapes={})
    for name, ms in runs.items():
        M, N, K = SHAPES[name][:3]
        med = statistics.median(m["ms"] for m in ms)
        shas = sorted({m["sha256"] for m in ms})
        res["shapes"][name] = dict(M=M, N=N, K=K, kernel=kernel_of(name), ms=med, ms_min=min(m["ms"] for m in ms),
                                   ms_max=max(m["ms"] for m in ms),
                                   tflops=(None if SHAPES[name][4] == "quant" else round(2 * M * N * K / (med * 1e-3) / 1e12, 1)),
                                   sha256=shas[0] if len(shas) == 1 else shas,
                                   cublas_tflops=ms[0].get("cublas_tflops"), sm_mhz=[m["sm_mhz"] for m in ms])
    ks = [(SHAPES[n][2], res["shapes"][n]["ms"]) for n in ("q_linear", "k2304", "k4608") if n in res["shapes"]]
    if len(ks) == 3:  # least-squares line of time against K at N 1152: the intercept is the per-tile cost the mainloop does not hide
        mk = sum(k for k, _ in ks) / 3
        mt = sum(t for _, t in ks) / 3
        slope = sum((k - mk) * (t - mt) for k, t in ks) / sum((k - mk) ** 2 for k, _ in ks)
        icpt = mt - slope * mk
        res["k_intercept"] = dict(ms=round(icpt, 4), ms_per_k1152=round(slope * 1152, 4),
                                  fraction_of_k1152=round(icpt / res["shapes"]["q_linear"]["ms"], 4))
        print(f"time vs K at N 1152: intercept {icpt:.4f} ms ({100 * icpt / res['shapes']['q_linear']['ms']:.1f} % of K 1152), "
              f"{slope * 1152:.4f} ms per 1152 of K", flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
