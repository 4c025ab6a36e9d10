"""ctypes binding of libmmx.so (C ABI declared in include/mmx.h).  There is no CPU fallback: if the library is
missing or a call fails, an exception is raised."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmmx.so")

c_float_p = C.c_void_p   # raw device / host pointers are passed as integers
c_int_p = C.c_void_p


class MmxError(RuntimeError):
    pass


class ClipConfigC(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "embed_dim", "image_resolution", "vision_layers", "vision_width", "vision_patch_size",
        "context_length", "vocab_size", "transformer_width", "transformer_heads", "transformer_layers")]


_SIGS = {
    "mmx_last_error": (C.c_char_p, []),
    "mmx_version": (C.c_int, []),
    "mmx_launch_count": (C.c_uint64, []),
    "mmx_set_gemm_backend": (C.c_int, [C.c_int]),
    "mmx_get_gemm_backend": (C.c_int, []),
    "mmx_set_gemm_tile_n": (C.c_int, [C.c_int]),
    "mmx_profile_gemm": (C.c_int, [C.c_int]),
    "mmx_profile_gemm_report": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    "mmx_gemm_trace": (C.c_int, [C.c_void_p]),
    "mmx_memcpy_d2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mmx_avg_heads": (C.c_int, [c_float_p, c_float_p, c_float_p] + [C.c_int] * 6 + [C.c_void_p]),
    "mmx_attn_gradcam": (C.c_int, [c_float_p, c_float_p, c_float_p, c_float_p] + [C.c_int] * 6 + [C.c_void_p]),
    "mmx_self_update": (C.c_int, [c_float_p, C.c_int, c_float_p, c_float_p, C.c_int, c_float_p, c_float_p, C.c_int,
                                  C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_self_chain": (C.c_int, [c_float_p, C.c_longlong, C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_handle_residual": (C.c_int, [c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, c_float_p, C.c_void_p]),
    "mmx_mm_update_workspace": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "mmx_mm_update": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int,
                                c_float_p, C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                C.c_void_p, c_float_p, C.c_void_p]),
    "mmx_rollout": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_float_p, c_float_p, C.c_void_p]),
    "mmx_minmax_normalize": (C.c_int, [c_float_p, c_float_p, C.c_int, C.c_longlong, C.c_void_p]),
    "mmx_otsu_masks": (C.c_int, [c_float_p, c_float_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "mmx_topk_select": (C.c_int, [c_float_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "mmx_bmm_add": (C.c_int, [c_float_p, C.c_int, C.c_longlong, C.c_int, c_float_p, C.c_int, C.c_longlong,
                              c_float_p, C.c_int, C.c_longlong, c_float_p, C.c_int, C.c_longlong,
                              C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_linear": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, c_float_p, C.c_int, c_float_p, C.c_int,
                             c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_linear_dgrad": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, C.c_int, c_float_p, C.c_int,
                                   C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_pack_weight_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "mmx_pack_weight": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "mmx_linear_packed": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, C.c_void_p, c_float_p, c_float_p, C.c_int, c_float_p,
                                    C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_linear_dgrad_packed": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, C.c_void_p, c_float_p, C.c_int, C.c_int,
                                          c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_gemm_nt": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, C.c_void_p, c_float_p, c_float_p, C.c_int, c_float_p, C.c_int,
                              c_float_p, C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_lrp_split": (C.c_int, [c_float_p, C.c_int, c_float_p, c_float_p, C.c_int, C.c_longlong, C.c_int, C.c_void_p]),
    "mmx_lrp_safe_divide": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, C.c_longlong, C.c_int, C.c_void_p]),
    "mmx_lrp_partials_len": (C.c_int, []),
    "mmx_lrp_sums": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "mmx_lrp_renorm": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mmx_lrp_add": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int,
                              C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "mmx_lrp_clone": (C.c_int, [c_float_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_int, c_float_p, C.c_int,
                                C.c_longlong, C.c_int, C.c_void_p]),
    "mmx_lrp_zero_value_fix": (C.c_int, [c_float_p, C.c_int, C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mmx_lrp_attn_pv": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p,
                                  c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_lrp_attn_qk": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, C.c_float, c_float_p, C.c_int,
                                  c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_lrp_attn_scores": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_float, c_float_p, c_float_p, C.c_int,
                                      C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_add": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, C.c_float, c_float_p, C.c_int, C.c_longlong, C.c_int, C.c_void_p]),
    "mmx_gather_rows": (C.c_int, [c_float_p, C.c_int, c_int_p, c_float_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_scatter_add_rows": (C.c_int, [c_float_p, C.c_int, c_int_p, c_float_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_act_bwd": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, C.c_int, c_float_p, C.c_int, C.c_longlong, C.c_int, C.c_void_p]),
    "mmx_act_fwd": (C.c_int, [c_float_p, C.c_int, C.c_int, c_float_p, C.c_int, C.c_longlong, C.c_int, C.c_void_p]),
    "mmx_im2col_patches": (C.c_int, [c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_layernorm_fwd": (C.c_int, [c_float_p, C.c_int, c_int_p, c_float_p, c_float_p, c_float_p, C.c_int, c_float_p,
                                    c_float_p, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "mmx_layernorm_bwd": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_int_p, c_float_p, c_float_p, c_float_p,
                                    c_float_p, C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_attention_fwd": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, c_float_p,
                                    C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                    C.c_int, C.c_void_p]),
    "mmx_attention_bwd": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int,
                                    c_float_p, c_float_p, C.c_int, c_float_p, c_float_p, C.c_int, c_float_p, C.c_int,
                                    c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int,
                                    C.c_void_p]),
    "mmx_attention_bwd_scaled": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int,
                                           c_float_p, c_float_p, C.c_int, c_float_p, c_float_p, C.c_int, c_float_p, C.c_int,
                                           c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int,
                                           c_float_p, C.c_void_p]),
    "mmx_attention_fwd_ragged": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int,
                                           c_float_p, C.c_int, c_int_p, c_int_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                           C.c_int, C.c_void_p]),
    "mmx_attention_bwd_ragged": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, C.c_int,
                                           c_float_p, c_float_p, C.c_int, c_float_p, c_float_p, C.c_int, c_float_p, C.c_int,
                                           c_float_p, C.c_int, c_int_p, c_int_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                           C.c_int, c_float_p, C.c_void_p]),
    "mmx_text_embed_packed": (C.c_int, [c_int_p, c_float_p, c_float_p, c_float_p, c_int_p, c_int_p, c_int_p, c_int_p,
                                        C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_vision_tokens_lnpre": (C.c_int, [c_float_p, C.c_int, c_float_p, c_float_p, c_float_p, c_float_p, c_float_p,
                                          C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "mmx_clip_head": (C.c_int, [c_float_p, c_float_p, C.c_float, c_float_p, c_float_p, c_float_p, c_float_p, c_float_p,
                                c_float_p, c_float_p, C.c_int, C.c_int, C.c_void_p]),
    "mmx_conv2d":(C.c_int, [c_float_p] + [C.c_longlong] * 4 + [C.c_int] * 4 + [c_float_p, C.c_int, C.c_void_p, c_float_p,
                                                                              c_float_p, C.c_int, c_float_p, C.c_int]
                   + [C.c_int] * 6 + [C.c_void_p]),
    "mmx_conv2d_dilated": (C.c_int, [c_float_p] + [C.c_longlong] * 4 + [C.c_int] * 4 + [c_float_p, C.c_int, C.c_void_p, c_float_p,
                                                                                      c_float_p, C.c_int, c_float_p, C.c_int]
                           + [C.c_int] * 7 + [C.c_void_p]),
    "mmx_maxpool2d_nhwc": (C.c_int, [c_float_p, C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mmx_detr_position_sine": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, c_float_p,
                                         C.c_int, C.c_void_p, C.c_void_p]),
    "mmx_detr_postprocess": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, c_float_p, C.c_void_p,
                                       C.c_void_p, c_float_p, C.c_void_p, c_float_p, C.c_void_p]),
    "mmx_detr_segm_postprocess": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int),
                                            C.POINTER(C.c_int), C.c_float, C.c_void_p, C.c_void_p]),
    "mmx_detr_match_cost": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p, c_float_p, C.POINTER(C.c_int), C.c_float, C.c_float, C.c_float, c_float_p,
                                      C.c_void_p, C.c_void_p]),
    "mmx_detr_match_lsa": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_void_p, C.c_void_p,
                                     C.c_void_p]),
    "mmx_detr_set_losses": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p, c_float_p, C.POINTER(C.c_int), C.c_void_p, c_float_p, c_float_p, c_float_p,
                                      C.c_void_p]),
    "mmx_detr_mask_losses": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p),
                                       C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.c_void_p, c_float_p, c_float_p,
                                       C.c_void_p]),
    "mmx_relevance_overlay": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, c_float_p, C.c_int,
                                        C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "mmx_box_relevance_image": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, c_float_p, c_float_p, C.c_int, C.c_int,
                                          C.c_void_p, C.c_void_p]),
    "mmx_clip_text_scores": (C.c_int, [c_float_p, c_int_p, C.c_int, C.c_int, c_float_p, c_int_p, C.c_void_p]),
    "mmx_clip_create": (C.c_int, [C.POINTER(ClipConfigC), C.c_int, C.POINTER(C.c_void_p)]),
    "mmx_clip_destroy": (None, [C.c_void_p]),
    "mmx_clip_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, c_float_p, C.c_size_t]),
    "mmx_clip_finalize": (C.c_int, [C.c_void_p]),
    "mmx_clip_set_serial": (C.c_int, [C.c_void_p, C.c_int]),
    "mmx_clip_interpret_device": (C.c_int, [C.c_void_p, c_float_p, C.c_int, c_int_p, C.c_int, C.c_int, C.c_int,
                                            c_float_p, c_float_p, C.c_void_p]),
    "mmx_clip_interpret_host": (C.c_int, [C.c_void_p, c_float_p, C.c_int, c_int_p, C.c_int, C.c_int, C.c_int,
                                          c_float_p, c_float_p]),
    "mmx_clip_tap": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int * 4),
                               C.POINTER(C.c_int)]),
}

_lib = None


def lib() -> C.CDLL:
    """Loads libmmx.so (once).  Raises MmxError if it has not been built - there is no fallback path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MmxError(f"{LIB_PATH} not found: build it with `python __graft_entry__.py` "
                           "(nvcc, sm_90a); the engine has no CPU / PyTorch fallback")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def exported_symbols():
    return sorted(_SIGS)


def check(rc: int):
    if rc != 0:
        raise MmxError(lib().mmx_last_error().decode("utf-8", "replace"))


def ptr(t):
    """device (or host) pointer of a torch tensor, or None."""
    return None if t is None else C.c_void_p(t.data_ptr())


def current_stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
