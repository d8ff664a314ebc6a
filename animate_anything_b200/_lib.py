"""ctypes binding of the C-ABI shared library `libaab200.so` (declared in include/aab200.h).

There is no CPU fallback: if the library is missing, or a kernel entry point returns a non-zero status, the product
path raises.  torch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("AAB_LIB_PATH") or os.path.join(_HERE, "libaab200.so")   # override: A/B builds while tuning

MAX_TAPS = 9
ACT_NONE, ACT_SILU, ACT_GELU, ACT_QUICK_GELU = 0, 1, 2, 3
F_BF16, F_DIRECT, F_OUT_F32, F_GEGLU, F_SCALE_ACC, F_TWO_CTA = 1, 2, 4, 8, 16, 64


class IgemmDesc(C.Structure):
    """Mirror of `AabIgemmDesc` (animate_anything_b200/csrc/igemm.h)."""

    _fields_ = [
        ("a", C.c_void_p), ("a_dims", C.c_long * 5), ("a_strides", C.c_long * 5),
        ("a2", C.c_void_p), ("a2_dims", C.c_long * 5), ("a2_strides", C.c_long * 5),
        ("kc", C.c_int), ("kc1", C.c_int), ("num_taps", C.c_int),
        ("tap_off", (C.c_int * 5) * MAX_TAPS),
        ("b", C.c_void_p), ("ld_b", C.c_long), ("b_batch", C.c_int), ("b_batch_stride", C.c_long),
        ("b_batch_dim", C.c_int), ("n", C.c_int),
        ("dim_d", C.c_int * 4), ("box", C.c_int * 4),
        ("out", C.c_void_p), ("ld_out", C.c_long),
        ("bias", C.c_void_p), ("bias2", C.c_void_p), ("rows_per_bias2", C.c_int), ("ld_bias2", C.c_long),
        ("residual", C.c_void_p), ("ld_res", C.c_long),
        ("out_scale", C.c_float), ("act", C.c_int), ("flags", C.c_int), ("block_n", C.c_int),
        ("colstats", C.c_void_p),
    ]


class AabError(RuntimeError):
    pass


_lib = None

_SIGS = {
    "aab_igemm": [C.POINTER(IgemmDesc), C.c_void_p],
    "aab_num_sms": [],
    "aab_flash_attn_d64": [C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_int,
                           C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_int, C.c_int,
                           C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                           C.c_float, C.c_int, C.c_void_p],
    "aab_flash_attn_d80": [C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_int,
                           C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_int, C.c_int,
                           C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                           C.c_float, C.c_int, C.c_void_p],
    "aab_clip_image_prep": [C.c_void_p, C.c_int, C.c_long, C.c_long, C.c_long, C.c_long, C.c_int, C.c_int, C.c_int,
                            C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_long,
                            C.c_int, C.c_void_p],
    "aab_temporal_attn_d64": [C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long, C.c_int, C.c_int,
                              C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p],
    "aab_groupnorm": [C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_long, C.c_int, C.c_long, C.c_long, C.c_int,
                      C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_void_p],
    "aab_groupnorm_colstats": [C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_long,
                               C.c_long, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_long, C.c_void_p,
                               C.c_int, C.c_void_p],
    "aab_layernorm": [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_float,
                      C.c_int, C.c_void_p],
    "aab_softmax_rows": [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_int, C.c_void_p],
    "aab_unet_in_assemble": [C.c_void_p, C.POINTER(C.c_long), C.c_void_p, C.POINTER(C.c_long), C.c_void_p,
                             C.POINTER(C.c_long), C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                             C.c_void_p],
    "aab_unet_out_finalize": [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_timestep_embed": [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_embed_tokens": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int,
                         C.c_void_p],
    "aab_image_to_nhwc16": [C.c_void_p, C.c_long, C.c_long, C.c_long, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_int,
                            C.c_int, C.c_int, C.c_void_p],
    "aab_add_rowvec": [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_long, C.c_int,
                       C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_axpby": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_float, C.c_float, C.c_int, C.c_void_p],
    "aab_svd_out_finalize": [C.c_void_p, C.c_int, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_svd_in_assemble": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                            C.c_int, C.c_int, C.c_void_p],
    "aab_svd_in_assemble_frames": [C.c_void_p, C.c_void_p, C.c_long, C.c_long, C.c_long, C.c_int, C.c_void_p, C.c_long, C.c_long,
                                   C.c_float, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_svd_cfg_euler_step": [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float,
                               C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_geglu": [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_int, C.c_void_p],
    "aab_upsample2x": [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_upsample_nearest": [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_pad_br": [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_copy2d": [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_long, C.c_int, C.c_void_p],
    "aab_dup_rows": [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p],
    "aab_transpose": [C.c_void_p, C.c_long, C.c_long, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_cfg_scheduler_step": [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_image_to_nhwc8": [C.c_void_p, C.c_long, C.c_long, C.c_long, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_int,
                           C.c_int, C.c_int, C.c_void_p],
    "aab_vae_enc_finalize": [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_int,
                             C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_vae_dec_in": [C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                       C.c_int, C.c_void_p],
    "aab_vae_dec_finalize": [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_vae_dec_finalize_u8": [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_add_noise": [C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_long,
                      C.c_int, C.c_void_p],
    "aab_cast_f32": [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_void_p],
    "aab_video_f32_to_nhwc8": [C.c_void_p, C.c_long, C.c_long, C.c_long, C.c_long, C.c_long, C.c_void_p, C.c_int, C.c_int,
                               C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p],
    "aab_rgba_finalize_u8": [C.c_void_p, C.c_int, C.c_void_p, C.c_long, C.c_int, C.c_void_p],
    "aab_pad_cols": [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_void_p],
}

EXPORTS = tuple(_SIGS.keys())

_launch_count = 0
_KERNELS_PER_CALL = {"aab_groupnorm": 2, "aab_groupnorm_colstats": 2}     # statistics + apply


def load():
    """dlopen libaab200.so; raises AabError if it has not been built (python __graft_entry__.py build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AabError(f"{LIB_PATH} not found: the CUDA extension is not built. Run `python __graft_entry__.py` "
                       f"(build()) or animate_anything_b200/csrc/build.sh. There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, args in _SIGS.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = C.c_int
    lib.aab_groupnorm_workspace_bytes.argtypes = [C.c_long, C.c_long, C.c_int, C.c_int]
    lib.aab_groupnorm_workspace_bytes.restype = C.c_long
    lib.aab_igemm_emits_colstats.argtypes = [C.POINTER(IgemmDesc)]
    lib.aab_igemm_emits_colstats.restype = C.c_int
    _lib = lib
    return lib


def call(name, *args):
    """Call a C-ABI entry point, raise on a non-zero status, count the launch."""
    global _launch_count
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise AabError(f"{name} failed with status {rc} (1=bad argument, 2=CUDA launch error, 3=driver/TMA encode)")
    _launch_count += _KERNELS_PER_CALL.get(name, 1)
    return rc


def launch_count() -> int:
    return _launch_count


def reset_launch_count():
    global _launch_count
    _launch_count = 0
