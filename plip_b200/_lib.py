"""ctypes binding of ``libplip_b200.so`` (the C ABI declared in ``include/plip_b200.h``).

The library is the only compute path of this package: if it is missing the import of
:func:`lib` raises — there is no CPU / PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libplip_b200.so"

_vp = C.c_void_p
_i = C.c_int
_i64 = C.c_int64
_u64 = C.c_uint64
_f = C.c_float
_fp = C.c_void_p  # float* passed as raw address


class TensorInfo(C.Structure):
    """Mirror of ``plip_tensor_info_t``."""

    _fields_ = [
        ("name", C.c_char * 96),
        ("offset", C.c_uint64),
        ("numel", C.c_uint64),
        ("dtype", C.c_int32),
        ("rows", C.c_int32),
        ("cols", C.c_int32),
        ("fused", C.c_int32),
    ]


class KernelTime(C.Structure):
    """Mirror of ``plip_kernel_time_t``."""

    _fields_ = [("name", C.c_char * 48), ("launches", C.c_int32), ("total_ms", C.c_float), ("flops", C.c_double),
                ("bytes", C.c_double)]


class ResizeDesc(C.Structure):
    """Mirror of ``plip_resize_desc_t`` (32 bytes; ``preprocess.RESIZE_DESC_DTYPE`` is the numpy twin)."""

    _fields_ = [
        ("offset", C.c_int64),
        ("width", C.c_int32),
        ("height", C.c_int32),
        ("new_width", C.c_int32),
        ("new_height", C.c_int32),
        ("left", C.c_int32),
        ("top", C.c_int32),
    ]


class SgdProblem(C.Structure):
    """Mirror of ``plip_sgd_problem_t`` (32 bytes)."""

    _fields_ = [("alpha", C.c_double), ("pos_weight", C.c_double), ("neg_weight", C.c_double), ("pos_class", C.c_int32),
                ("sigma_index", C.c_int32)]


class TowerOutputs(C.Structure):
    """Mirror of ``plip_tower_outputs_t`` (device pointers, 0 = not requested)."""

    _fields_ = [("embeds", C.c_void_p), ("pooled", C.c_void_p), ("last_hidden", C.c_void_p), ("hidden", C.c_void_p),
                ("attn", C.c_void_p), ("normalize", C.c_int32)]


# name -> (restype, argtypes); must list every PLIP_API symbol of include/plip_b200.h
SIGNATURES = {
    "plip_last_error": (C.c_char_p, []),
    "plip_abi_version": (_i, []),
    "plip_launch_count": (_u64, []),
    "plip_weights_num_tensors": (_i, []),
    "plip_weights_tensor_info": (_i, [_i, C.POINTER(TensorInfo)]),
    "plip_weights_blob_bytes": (_u64, []),
    "plip_create": (_i, [_vp, _u64, _f, _i, _i, C.POINTER(_vp)]),
    "plip_create_ex": (_i, [_vp, _u64, _f, _i, _i, _i, C.POINTER(_vp)]),
    "plip_operand_format": (_i, [_vp]),
    "plip_set_text_pooling": (_i, [_vp, _i]),
    "plip_set_last_layer_pruning": (_i, [_vp, _i]),
    "plip_last_layer_pruning": (_i, [_vp]),
    "plip_dbg_set_operand_format": (_i, [_i]),
    "plip_destroy": (_i, [_vp]),
    "plip_workspace_bytes": (_u64, [_i]),
    "plip_logit_scale_exp": (_f, [_vp]),
    "plip_max_micro_batch": (_i, [_vp]),
    "plip_encode_images": (_i, [_vp, _vp, _i, _i64, _fp, _i, _vp]),
    "plip_encode_images_hw": (_i, [_vp, _vp, _i, _i64, _i, _i, _fp, _i, _vp]),
    "plip_encode_windows": (_i, [_vp, _vp, _i, _i, _i64, _vp, _i64, _fp, _i, _vp]),
    "plip_window_background_counts": (_i, [_vp, _i, _i, _i64, _vp, _i64, _i, _vp, _vp]),
    "plip_encode_text": (_i, [_vp, _vp, _i, _vp, _i64, _i, _fp, _i, _vp]),
    "plip_encode_text_prefix": (_i, [_vp, _vp, _i, _vp, _i64, _i, _i, _fp, _i, _vp]),
    "plip_vision_outputs": (_i, [_vp, _vp, _i, _i64, _i, _i, C.POINTER(TowerOutputs), _vp]),
    "plip_text_outputs": (_i, [_vp, _vp, _i, _vp, _i64, _i, C.POINTER(TowerOutputs), _vp]),
    "plip_similarity": (_i, [_fp, _i64, _fp, _i64, _f, _i, _i, _fp, _i64, _vp]),
    "plip_similarity_topk": (_i, [_fp, _i64, _fp, _i64, _f, _i, _i, _i, _vp, _fp, _vp]),
    "plip_l2_normalize": (_i, [_fp, _i64, _i, _vp]),
    "plip_window_mask_counts": (_i, [_vp, _i, _i, _i, _i64, _vp, _i64, _i, _vp, _vp]),
    "plip_resize_crop_u8": (_i, [_vp, _u64, _vp, _i64, _vp, _vp]),
    "plip_resize_crop_bilinear_u8": (_i, [_vp, _u64, _vp, _i64, _vp, _vp]),
    "plip_resize_region_workspace": (_i, [_i, _i, _i, _i, _i, _i, C.POINTER(_u64)]),
    "plip_resize_region_u8": (_i, [_vp, _i64, _i, _i, _i, _i, _vp, _i64, _i, _i, _i, _i, _vp, _u64, _vp]),
    "plip_resize_filter_bounds": (_i, [_i, _i, _vp]),
    "plip_sgd_shuffle_permutation": (_i, [_i64, C.c_uint32, _vp]),
    "plip_sgd_workspace_bytes": (_i, [_i64, _i, _i, C.POINTER(_u64)]),
    "plip_sgd_fit": (_i, [_fp, _i64, _i, _vp, _i, _vp, _i, _vp, _i, _i, C.c_double, _i, _fp, _vp, _vp, _vp, _vp, _u64,
                          _vp]),
    "plip_linear_decision": (_i, [_fp, _i64, _i, _fp, _vp, _i, _fp, _vp, _vp]),
    "plip_densenet_num_tensors": (_i, []),
    "plip_densenet_tensor_info": (_i, [_i, C.POINTER(TensorInfo)]),
    "plip_densenet_blob_bytes": (_u64, []),
    "plip_densenet_workspace_bytes": (_u64, [_i]),
    "plip_densenet_create": (_i, [_vp, _u64, _i, _i, C.POINTER(_vp)]),
    "plip_densenet_destroy": (_i, [_vp]),
    "plip_densenet_max_micro_batch": (_i, [_vp]),
    "plip_densenet_encode": (_i, [_vp, _vp, _i64, _fp, _vp]),
    "plip_encode_images_host": (_i, [_vp, _vp, _i, _i64, _fp, _i]),
    "plip_encode_text_host": (_i, [_vp, _vp, _i, _vp, _i64, _i, _fp, _i]),
    "plip_profile_enable": (_i, [_vp, _i]),
    "plip_profile_read": (_i, [_vp, C.POINTER(KernelTime), _i, C.POINTER(_i)]),
    "plip_dbg_gemm": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _fp, _vp, _i, _fp, _i, _i, _i, _fp, _fp, _i, _vp, _fp, _vp]),
    "plip_dbg_resize_filter": (_i, [_i, _i, _i, _vp, _i, C.POINTER(_i), C.POINTER(_i)]),
    "plip_dbg_resize_filter_bilinear": (_i, [_i, _i, _i, _vp, _i, C.POINTER(_i), C.POINTER(_i)]),
    "plip_dbg_text_bucket_plan": (_i, [_vp, _i64, _i, _vp, _vp, _vp, _i]),
    "plip_dbg_rowstats_cast": (_i, [_fp, _i64, _i, _vp, _fp, _vp]),
    "plip_dbg_layernorm": (_i, [_fp, _i64, _i, _i64, _fp, _fp, _fp, _vp, _vp]),
    "plip_dbg_attention": (_i, [_vp, _i64, _i, _i, _i, _vp, _vp, _vp]),
    "plip_dbg_attention_probs": (_i, [_vp, _i64, _i, _i, _i, _vp, _fp, _vp]),
    "plip_dbg_densenet_op": (_i, [_i, _vp, _i, _i64, _i, _i, _vp, _fp, _fp, _fp, _fp, _vp, _i, _vp]),
    "plip_dbg_im2col": (_i, [_vp, _i, _i64, _vp, _vp]),
    "plip_dbg_hidden_states": (_i, [_vp, _i, _vp, _i, _vp, _i64, _i, _fp, _vp]),
    "plip_dbg_pos_interp": (_i, [_fp, _i, _i, _fp, _vp]),
    "plip_dbg_hidden_states_hw": (_i, [_vp, _vp, _i, _i64, _i, _i, _i, _fp, _vp]),
}

_LIB = None


def lib(strict: bool = True) -> C.CDLL:
    """Load the CUDA library (once).  ``strict`` requires every declared symbol to be exported."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m plip_b200.build` "
            "(plip_b200 has no CPU fallback; the sm_90a CUDA library is the product)."
        )
    dll = C.CDLL(str(LIB_PATH))
    missing = []
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(dll, name)
        except AttributeError:
            missing.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    if missing and strict:
        raise RuntimeError(f"{LIB_PATH} does not export: {missing}")
    _LIB = dll
    return dll


def last_error() -> str:
    msg = lib(strict=False).plip_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed (rc={rc}): {last_error()}")
