"""ctypes binding of libvideoswap_b200.so (the C-ABI in include/videoswap_b200.h).

There is NO fallback: if the shared library is missing or a call fails, an exception is raised.  The library is
built in-tree by `python -m videoswap_b200.build` / `__graft_entry__.build()`.
"""
from __future__ import annotations

import ctypes as C
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libvideoswap_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(HERE), "include", "videoswap_b200.h")


class VSError(RuntimeError):
    pass


class UNetConfigStruct(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int), ("out_channels", C.c_int), ("block_out_channels", C.c_int * 4),
        ("layers_per_block", C.c_int), ("num_heads", C.c_int), ("cross_attention_dim", C.c_int),
        ("norm_num_groups", C.c_int), ("norm_eps", C.c_float), ("use_motion_module", C.c_int),
        ("motion_down", C.c_int * 4), ("motion_up", C.c_int * 4), ("motion_mid", C.c_int),
        ("motion_num_heads", C.c_int), ("pe_max_len", C.c_int),
    ]


_P = C.c_void_p
_I = C.c_int
_F = C.c_float
_LL = C.c_longlong
_SZ = C.c_size_t

_SIGNATURES = {
    "vs_last_error": (C.c_char_p, []),
    "vs_version": (_I, []),
    "vs_unet_create": (_I, [C.POINTER(UNetConfigStruct), C.POINTER(_P)]),
    "vs_unet_destroy": (None, [_P]),
    "vs_unet_load_weights": (_I, [_P, _P, _I, C.POINTER(C.c_char_p), C.POINTER(_P), C.POINTER(C.c_int64)]),
    "vs_unet_num_params": (_I, [_P]),
    "vs_unet_param_name": (C.c_char_p, [_P, _I]),
    "vs_unet_forward": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _I, C.POINTER(_P), _I, _F, _P]),
    "vs_unet_workspace_bytes": (_SZ, [_P]),
    "vs_unet_pin_workspace": (_I, [_P, _I]),
    "vs_unet_reserve_workspace": (_I, [_P, _I, _I, _I, _I]),
    "vs_comm_unique_id": (_I, [_P]),
    "vs_comm_create": (_I, [_P, _I, _I, C.POINTER(_P)]),
    "vs_comm_destroy": (None, [_P]),
    "vs_comm_all_gather": (_I, [_P, _P, _P, _P, _SZ]),
    "vs_comm_all_reduce_sum_f32": (_I, [_P, _P, _P, _SZ]),
    "vs_unet_set_frame_shard": (_I, [_P, _P, _I, _I]),
    "vs_unet_enable_taps": (_I, [_P, _I]),
    "vs_unet_num_taps": (_I, [_P]),
    "vs_unet_get_tap": (_I, [_P, _I, C.POINTER(C.c_char_p), C.POINTER(_P), C.POINTER(_I), C.POINTER(_I), C.POINTER(_I),
                             C.POINTER(_I)]),
    "vs_unet_copy_tap": (_I, [_P, _P, _I, _P]),
    "vs_profile_enable": (_I, [_I]),
    "vs_profile_reset": (_I, []),
    "vs_profile_collect": (_I, [_I, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_longlong)]),
    "vs_launch_count": (C.c_longlong, []),
    "vs_set_option": (_I, [C.c_char_p, _I]),
    "vs_profile_dump": (_I, [C.c_char_p]),
    "vs_cfg_ddim_step": (_I, [_P, _P, _P, _I, _SZ, _I, _F, _F, _F, _P]),
    "vs_cfg_ddim_step_dev": (_I, [_P, _P, _P, _I, _SZ, _I, _F, _P, _P]),
    "vs_adapter_level": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _I, _I, _I, _I, _F, _I, _F, _P, _P]),
    "vs_gemm": (_I, [_P, _P, _I, _P, _I, _P, _I, _I, _P, _P, _I, _P, _P, _I, _I]),
    "vs_conv3x3": (_I, [_P, _P, _I, _P, _I, _P, _I, _I, _I, _I, _P, _P, _I, _P, _P]),
    "vs_pack_conv3x3": (_I, [_P, _P, _I, _I, _P]),
    "vs_pack_geglu": (_I, [_P, _P, _P, _I, _I, _P, _P]),
    "vs_groupnorm": (_I, [_P, _P, _I, _P, _I, _I, _I, _I, _I, _F, _P, _P, _I, _P, _P]),
    "vs_layernorm": (_I, [_P, _P, _I, _I, _P, _P, _P, _I, _I, _P]),
    "vs_ln_linear": (_I, [_P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "vs_unet_set_attention_hook": (_I, [_P, _P, _P, _I]),      # hook: CFUNCTYPE object or None
    "vs_attention_probs": (_I, [_P, _P, _I, _P, _I, _P, _I, _I, _I, _I, _I, _LL, _LL, _I]),
    "vs_attention_apply_probs": (_I, [_P, _P, _P, _I, _P, _I, _I, _I, _I, _I, _I, _LL, _LL, _I]),
    "vs_blend_mask": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _I, _I, _I, _F, _I, _P]),
    "vs_latent_blend": (_I, [_P, _P, _P, _P, _I, _I, _I, _I]),
    "vs_linear_ln_linear": (_I, [_P, _P, _I, _I, _P, _P, _P, _I, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _I, _P]),
    "vs_attention": (_I, [_P, _P, _I, _P, _I, _P, _I, _P, _I, _I, _I, _I, _I, _I, _LL, _LL, _LL, _I]),
    "vs_temporal_attention": (_I, [_P, _P, _P, _I, _I, _I, _I, _I]),
    "vs_conv_in": (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _I, _P]),
    "vs_upsample2x": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "vs_upsample_conv3x3": (_I, [_P, _P, _I, _I, _I, _I, _P, _I, _P, _P, _P]),
    "vs_conv3x3_s2": (_I, [_P, _P, _I, _I, _I, _I, _P, _I, _P, _P, _P]),
}

_lib = None


def header_symbols():
    """Every function name declared in include/videoswap_b200.h."""
    with open(HEADER_PATH) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(vs_[a-z0-9_]+)\s*\(", text)))


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VSError(f"{LIB_PATH} is missing: build it with `python -m videoswap_b200.build` "
                          f"(there is no CPU/PyTorch fallback for this path)")
        _lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype = res
            fn.argtypes = args
    return _lib


def check(code: int, what: str = ""):
    if code != 0:
        msg = lib().vs_last_error()
        raise VSError(f"{what or 'videoswap_b200 call'} failed ({code}): {msg.decode() if msg else '?'}")


def call(name: str, *args):
    """Calls an int-returning entry point and raises on error."""
    check(getattr(lib(), name)(*args), name)
