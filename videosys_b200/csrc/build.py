"""Builds libvsb200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m videosys_b200.csrc.build [--force] [--verbose]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["api.cu", "elementwise.cu", "attn_short.cu", "gemm_wgmma.cu", "attn_wgmma.cu", "attn_mma.cu", "dsp_p2p.cu", "patch_embed.cu", "dwconv.cu", "vae_conv.cu", "vae_osp.cu"]
# every kernel file below is compiled twice: bf16 (as is) and IEEE fp16 (-DVSB_HALF -> *.f16.o, entries suffixed _f16)
TWINNED = ["elementwise.cu", "attn_short.cu", "gemm_wgmma.cu", "attn_wgmma.cu", "attn_mma.cu", "patch_embed.cu", "dwconv.cu", "vae_conv.cu", "vae_osp.cu"]
HEADERS = ["vsb_common.cuh", "vsb_host.h", "wgmma.cuh", "attn_params.cuh", "dsp_common.cuh", os.path.join("..", "..", "include", "vsb200.h")]
LIB = os.path.join(HERE, "libvsb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _stale(obj, src):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    # this file too: a change of FLAGS (the target architecture) must rebuild every object
    deps = [src, os.path.abspath(__file__)] + [os.path.join(HERE, h) for h in HEADERS]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    objs = []
    procs = []
    jobs = [(s, s.replace(".cu", ".o"), []) for s in SOURCES] + [(s, s.replace(".cu", ".f16.o"), ["-DVSB_HALF"]) for s in TWINNED]
    for s, o, extra in jobs:
        src = os.path.join(HERE, s)
        obj = os.path.join(HERE, o)
        objs.append(obj)
        if force or _stale(obj, src):
            cmd = [NVCC, *FLAGS, *extra, "-c", src, "-o", obj]
            procs.append((o, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            print(f"[vsb200 build] {s} FAILED\n{out}", file=sys.stderr)
        elif verbose:
            print(f"[vsb200 build] {s}\n{out}")
    if failed:
        raise RuntimeError("nvcc failed")
    if procs or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB, *objs, "-lcudart"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
