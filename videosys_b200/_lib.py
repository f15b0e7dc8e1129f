"""ctypes binding of libvsb200.so (the C-ABI declared in include/vsb200.h).

The library is built in-tree by ``videosys_b200.csrc.build`` (nvcc, sm_90a).  There is no CPU path and
no alternative backend: if the shared object is missing and cannot be built, importing the kernels fails.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libvsb200.so")

_vp, _i, _ll, _f, _sz, _u = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_size_t, C.c_uint

# name -> (restype, argtypes); must list every symbol include/vsb200.h declares (tests/test_host_cpu.py::test_library_exports_every_declared_symbol checks)
SIGNATURES = {
    "vsb_version": (_i, []),
    "vsb_last_error": (C.c_char_p, []),
    "vsb_init": (_i, [_i]),
    "vsb_launch_count": (C.c_ulonglong, []),
    "vsb_set_option": (_i, [C.c_char_p, _i]),
    "vsb_ln_modulate": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "vsb_ln_modulate_affine": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "vsb_qk_layernorm": (_i, [_vp, _vp, _vp, _vp, _vp, _sz, _i, _i, _f, _vp]),
    "vsb_modulation_table": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "vsb_gate_residual": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "vsb_residual_add": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "vsb_qk_rmsnorm": (_i, [_vp, _vp, _vp, _sz, _i, _i, _f, _vp]),
    "vsb_attn_short": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _ll, _ll, _ll, _i, _i, _i, _f, _f, _i, _vp]),
    "vsb_gemm_bias_act": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "vsb_gemm_bias_residual": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_gemm_kernel_name": (C.c_char_p, [_i, _i, _i, _i, _i]),
    "vsb_quant_rows_fp8": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "vsb_ln_modulate_fp8": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "vsb_gemm_fp8_bias_act": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "vsb_gemm_fp8_bias_residual": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_gemm_fp8_kernel_name": (C.c_char_p, [_i, _i, _i, _i, _i]),
    "vsb_attn_flash": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _ll, _ll, _ll, _ll, C.POINTER(_i), _f, _vp]),
    "vsb_pab_gate": (_i, [_i, _i, _i, C.POINTER(_i), _i, _i, _i, _i]),
    "vsb_dsp_wait": (_i, [_vp, _i, _u, _vp]),
    "vsb_dsp_signal": (_i, [C.POINTER(_vp), _i, _i, _u, _vp]),
    "vsb_ln_modulate_dsp": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, C.POINTER(_vp), C.POINTER(_vp), _i, _i, _i, _u,
                                _vp]),
    "vsb_gate_residual_dsp": (_i, [_vp, C.POINTER(_vp), _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_qk_rmsnorm_rope": (_i, [_vp, _vp, _vp, _sz, _i, _i, _f, _vp, _vp, _i, _i, _vp]),
    "vsb_qk_rope_halves": (_i, [_vp, _sz, _i, _i, _i, _vp, _vp, _i, _i, _vp]),
    "vsb_attn_flash_strided": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _ll, _ll, _ll, _ll, _ll, _ll, C.POINTER(_i), _f,
                                   _vp]),
    "vsb_patch_embed": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _ll, _ll, _ll, _i, _i, _i, _i, _i, _vp]),
    "vsb_dwconv_shuffle": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_gate_residual_unshuffle": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_dwconv_ffn": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "vsb_kv_compress": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _f, _i, _vp]),
    "vsb_vae_conv3d": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_vae_groupnorm_stats": (_i, [_vp, _vp, _vp, _i, _ll, _i, _i, _f, _vp]),
    "vsb_vae_spatial_norm_silu": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_vae_upsample2x": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_vae_groupnorm_act": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_vae_upsample_linear2x": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_vae_mix": (_i, [_vp, _vp, _vp, _i, _i, _ll, _i, _i, _f, _f, _vp]),
    "vsb_vae_attn_split": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_vae_attn_softmax": (_i, [_vp, _i, _i, _i, _f, _vp]),
    "vsb_vae_attn_merge": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "vsb_vae_depth_to_time": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_vae_conv_time": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _f, _f, _i, _vp]),
    "vsb_vae_time_conv_rgb": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "vsb_vae_conv_down": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "vsb_tmap_cache_stats": (C.c_ulonglong, [_i]),
    "vsb_dsp_alloc": (_i, [C.POINTER(_vp), _sz]),
    "vsb_dsp_free": (_i, [_vp]),
    "vsb_ipc_get_handle": (_i, [_vp, _vp]),
    "vsb_ipc_open_handle": (_i, [_vp, C.POINTER(_vp)]),
    "vsb_ipc_close_handle": (_i, [_vp]),
}

# fp16 twins (include/vsb200.h "IEEE fp16 twins"): same signatures, suffix _f16
F16_TWINS = ("vsb_ln_modulate", "vsb_ln_modulate_affine", "vsb_modulation_table", "vsb_gate_residual", "vsb_residual_add",
             "vsb_qk_rmsnorm", "vsb_qk_rmsnorm_rope", "vsb_qk_rope_halves", "vsb_qk_layernorm", "vsb_attn_short", "vsb_gemm_bias_act",
             "vsb_gemm_bias_residual", "vsb_quant_rows_fp8", "vsb_ln_modulate_fp8", "vsb_gemm_fp8_bias_act",
             "vsb_gemm_fp8_bias_residual", "vsb_attn_flash", "vsb_attn_flash_strided", "vsb_patch_embed",
             "vsb_dwconv_shuffle", "vsb_gate_residual_unshuffle", "vsb_dwconv_ffn", "vsb_kv_compress",
             "vsb_vae_conv3d", "vsb_vae_groupnorm_stats", "vsb_vae_spatial_norm_silu", "vsb_vae_upsample2x",
             "vsb_vae_groupnorm_act", "vsb_vae_upsample_linear2x", "vsb_vae_mix", "vsb_vae_attn_split", "vsb_vae_attn_softmax",
             "vsb_vae_attn_merge", "vsb_vae_depth_to_time", "vsb_vae_conv_time", "vsb_vae_time_conv_rgb",
             "vsb_vae_conv_down")
for _n in F16_TWINS:
    SIGNATURES[_n + "_f16"] = SIGNATURES[_n]

_lib = None


def load(build_if_missing: bool = True):
    """Returns the loaded library (cached).  Raises if it cannot be found or built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if not build_if_missing:
            raise RuntimeError(f"{LIB_PATH} missing: run `python -m videosys_b200.csrc.build`")
        from .csrc.build import build

        build()
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header / library drift
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class VsbError(RuntimeError):
    pass


def check(rc: int, what: str = ""):
    if rc < 0:
        msg = load().vsb_last_error().decode(errors="replace")
        raise VsbError(f"vsb200 {what} failed (status {rc}): {msg}")
    return rc
