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


class ImlpDescStruct(C.Structure):
    """vs_imlp_desc: one IMLP_Hash network (see the header)."""
    _fields_ = [("params", _P), ("input_dim", _I), ("output_dim", _I), ("hidden_dim", _I), ("mlp_layers", _I),
                ("pe_dim", _I), ("skip_mask", C.c_uint32), ("use_tanh", _I)]


class GemmDescStruct(C.Structure):
    """vs_gemm_desc: one launch of the tensor-core GEMM / implicit-GEMM convolution (see the header)."""
    _fields_ = [
        ("A", _P), ("K1", _I), ("lda1", _I),
        ("A2", _P), ("K2", _I), ("lda2", _I),
        ("Bw", _P),
        ("M", _I), ("N", _I),
        ("taps", _I),
        ("sub_py", _I), ("sub_px", _I),
        ("nimg", _I), ("H", _I), ("W", _I),
        ("bias", _P),
        ("rowvec", _P), ("ldrv", _I), ("pix_per_batch", _I), ("rv_mod", _I),
        ("ln_stats", _P), ("ln_u", _P),
        ("ln_parts", _P), ("ln_nparts", _I),
        ("ln_sums_out", _P),
        ("residual", _P), ("ldr", _I),
        ("out", _P), ("ldc", _I),
        ("mode", _I),
        ("force_bn", _I),
        ("OH", _I), ("OW", _I),
        ("stride2", _I),
    ]

_SIGNATURES = {
    "vs_last_error": (C.c_char_p, []),
    "vs_version": (_I, []),
    "vs_unet_create": (_I, [C.POINTER(UNetConfigStruct), C.POINTER(_P)]),
    "vs_unet_destroy": (None, [_P]),
    "vs_unet_load_weights": (_I, [_P, _P, _I, C.POINTER(C.c_char_p), C.POINTER(_P), C.POINTER(C.c_int64)]),
    "vs_unet_num_params": (_I, [_P]),
    "vs_unet_param_name": (C.c_char_p, [_P, _I]),
    "vs_unet_forward": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _I, C.POINTER(_P), _I, _F, _P]),
    "vs_unet_time_embedding": (_I, [_P, _P, _P, _I, _P, _P]),
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
    "vs_cfg_ddim_rescale_step": (_I, [_P, _P, _P, _P, _I, _I, _SZ, _I, _F, _F, _F, _F, _F, _P]),
    "vs_cfg_ddim_rescale_step_dev": (_I, [_P, _P, _P, _P, _I, _I, _SZ, _I, _F, _P, _P]),
    "vs_adapter_level": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _I, _I, _I, _I, _F, _I, _F, _P, _P]),
    "vs_gemm_ex": (_I, [_P, C.POINTER(GemmDescStruct)]),
    "vs_pack_conv3x3": (_I, [_P, _P, _I, _I, _P]),
    "vs_pack_geglu": (_I, [_P, _P, _P, _I, _I, _P, _P]),
    "vs_groupnorm": (_I, [_P, _P, _I, _P, _I, _I, _I, _I, _I, _F, _P, _P, _I, _P, _P]),
    "vs_groupnorm_stats": (_I, [_P, _P, _I, _P, _I, _I, _I, _I, _I, _P, _I]),
    "vs_groupnorm_apply": (_I, [_P, _P, _I, _P, _I, _I, _I, _I, _I, _P, _F, _P, _P, _I, _I, _P]),
    "vs_layernorm": (_I, [_P, _P, _I, _I, _P, _P, _P, _I, _I, _P]),
    "vs_ln_linear": (_I, [_P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "vs_unet_set_attention_hook": (_I, [_P, _P, _P, _I]),      # hook: CFUNCTYPE object or None
    "vs_attention_probs": (_I, [_P, _P, _I, _P, _I, _P, _I, _I, _I, _I, _I, _LL, _LL, _I]),
    "vs_attention_apply_probs": (_I, [_P, _P, _P, _I, _P, _I, _I, _I, _I, _I, _I, _LL, _LL, _I]),
    "vs_blend_mask": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _I, _I, _I, _F, _I, _P]),
    "vs_latent_blend": (_I, [_P, _P, _P, _P, _I, _I, _I, _I]),
    "vs_linear_ln_linear": (_I, [_P, _P, _I, _I, _P, _P, _P, _I, _P, _P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P,
                                 _P, _I, _P]),
    "vs_attention": (_I, [_P, _P, _I, _P, _I, _P, _I, _P, _I, _I, _I, _I, _I, _I, _LL, _LL, _LL, _I]),
    "vs_temporal_attention": (_I, [_P, _P, _P, _I, _I, _I, _I, _I]),
    "vs_conv_in": (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _I, _P, _P]),
    "vs_upsample2x": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "vs_upsample_conv3x3": (_I, [_P, _P, _I, _I, _I, _I, _P, _I, _P, _P, _P]),
    "vs_upsample_conv3x3_sized": (_I, [_P, _P, _I, _I, _I, _I, _P, _I, _P, _I, _I, _P, _P]),
    "vs_upsample_nearest": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "vs_conv3x3_s2": (_I, [_P, _P, _I, _I, _I, _I, _P, _I, _P, _P, _P]),
    "vs_pack_conv_subpixel": (_I, [_P, _P, _I, _I, _P]),
    "vs_softmax_rows": (_I, [_P, _P, _I, _I, _I, _F]),
    "vs_transpose_pad": (_I, [_P, _P, _I, _I, _I, _P]),
    "vs_vae_latent_in": (_I, [_P, _P, _I, _I, _I, _I, _F, _P, _P]),
    "vs_image_postprocess": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "vs_downsample_conv3x3": (_I, [_P, _P, _I, _I, _I, _I, _P, _I, _P, _P]),
    "vs_vae_image_in": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "vs_vae_moments": (_I, [_P, _P, _I, _I, _I, _P, _P]),
    "vs_t2i_image_in": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "vs_avgpool2x2": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "vs_scale_f16": (_I, [_P, _P, _SZ, _F, _P]),
    "vs_vae_posterior": (_I, [_P, _P, _P, _I, _I, _I, _F, _I, _P]),
    "vs_clip_embed": (_I, [_P, _P, _I, _I, _P, _I, _P, _I, _P]),
    "vs_causal_attention": (_I, [_P, _P, _I, _P, _I, _I, _I, _I, _I]),
    "vs_unet_forward_features": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _I, _I, _P]),
    "vs_dift_noise": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _F, _F, _P]),
    "vs_dift_point_sample": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _I, _P]),
    "vs_dift_ensemble_mean": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "vs_dift_point_reduce": (_I, [_P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    "vs_imlp_forward": (_I, [_P, C.POINTER(ImlpDescStruct), _P, _I, _P]),
    "vs_atlas_propagate": (_I, [_P, C.POINTER(ImlpDescStruct), C.POINTER(ImlpDescStruct), C.POINTER(ImlpDescStruct), _P, _F,
                                _I, _I, _I, _P, _P]),
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
