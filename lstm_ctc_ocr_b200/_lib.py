"""ctypes binding of libcrnnctc.so (include/crnn_ctc.h).  No CPU fallback: a missing or
unloadable library raises immediately."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcrnnctc.so")

c_int, c_float, c_size_t, c_void_p, c_char_p, c_int64 = (ctypes.c_int, ctypes.c_float, ctypes.c_size_t,
                                                         ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int64)


class CrnnConfig(ctypes.Structure):
    _fields_ = [("img_height", c_int), ("nclasses", c_int), ("num_hid", c_int), ("bn_eps", c_float),
                ("weight_decay", c_float), ("compute_dtype", c_int)]


# name -> (restype, argtypes); mirrors include/crnn_ctc.h one to one
SIGNATURES = {
    "crnn_version": (c_int, []),
    "crnn_status_string": (c_char_p, [c_int]),
    "crnn_last_error": (c_char_p, []),
    "crnn_ctc_workspace_size": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "crnn_ctc_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                              c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    "crnn_ctc_align_workspace_size": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "crnn_ctc_align": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                               c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "crnn_lexicon_candidates": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                        c_void_p, c_void_p, c_void_p]),
    "crnn_ctc_lexicon_score": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                       c_void_p, c_void_p, c_void_p, c_void_p]),
    "crnn_resize_lines_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "crnn_png_plan": (c_int, [c_void_p, c_void_p, c_int, c_void_p, ctypes.POINTER(c_size_t)]),
    "crnn_png_decode_gray_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_size_t, c_void_p]),
    "crnn_jpeg_plan": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, ctypes.POINTER(c_size_t)]),
    "crnn_jpeg_decode_gray_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_size_t, c_void_p]),
    "crnn_render_layout": (c_int, [c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "crnn_render_workspace_size": (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "crnn_render_lines_u8": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "crnn_ctc_greedy": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "crnn_ctc_beam_search": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int]),
    "crnn_ctc_beam_workspace_size": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "crnn_ctc_beam_search_device": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_size_t, c_void_p]),
    "crnn_ctc_beam_search_topk": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_int]),
    "crnn_ctc_beam_search_topk_device": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                                 c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "crnn_host_is_pinned": (c_int, [c_void_p]),
    "crnn_model_create": (c_int, [ctypes.POINTER(CrnnConfig), ctypes.POINTER(c_void_p)]),
    "crnn_model_destroy": (c_int, [c_void_p]),
    "crnn_num_tensors": (c_int, [c_void_p]),
    "crnn_param_count": (c_int64, [c_void_p]),
    "crnn_param_info": (c_int, [c_void_p, c_int, ctypes.POINTER(c_char_p), ctypes.POINTER(c_int64),
                                ctypes.POINTER(c_int64 * 4), ctypes.POINTER(c_int)]),
    "crnn_model_bind": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "crnn_model_params_changed": (c_int, [c_void_p]),
    "crnn_model_workspace_size": (c_int, [c_void_p, c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "crnn_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "crnn_forward_host": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t, c_int,
                                  c_void_p, c_void_p]),
    "crnn_forward_pageable": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t, c_int,
                                      c_int, c_void_p, c_void_p]),
    "crnn_lines_workspace_size": (c_int, [c_void_p, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "crnn_forward_lines": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "crnn_model_calibrate_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    # uint8 twins: the same arguments, uint8 pixels in place of the f32 data
    "crnn_forward_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "crnn_forward_host_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t, c_int,
                                     c_void_p, c_void_p]),
    "crnn_forward_pageable_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t,
                                         c_int, c_int, c_void_p, c_void_p]),
    "crnn_forward_lines_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "crnn_model_calibrate_fp8_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "crnn_backward_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "crnn_model_get_fp8_scales": (c_int, [c_void_p, c_void_p]),
    "crnn_model_set_fp8_scales": (c_int, [c_void_p, c_void_p]),
    "crnn_model_bind_bn_moving": (c_int, [c_void_p, c_void_p, c_float]),
    "crnn_model_set_bn_statistics": (c_int, [c_void_p, c_int]),
    "crnn_host_copy": (c_int, [c_void_p, c_void_p, c_size_t, c_int]),
    "crnn_total_loss": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "crnn_debug_tap": (c_int, [c_void_p, c_char_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "crnn_debug_tap_raw": (c_int, [c_void_p, c_char_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "crnn_profile_begin": (c_int, [c_void_p, c_int]),
    "crnn_profile_num_stages": (c_int, []),
    "crnn_profile_stage_name": (c_char_p, [c_int]),
    "crnn_profile_read": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int)]),
    "crnn_profile_bwd_num_stages": (c_int, []),
    "crnn_profile_bwd_stage_name": (c_char_p, [c_int]),
    "crnn_profile_bwd_read": (c_int, [c_void_p, c_void_p, ctypes.POINTER(c_int)]),
    "crnn_model_set_training": (c_int, [c_void_p, c_int]),
    "crnn_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "crnn_clip_adam_step": (c_int, [c_void_p, c_float, c_float, c_int, c_float, c_float, c_void_p]),
    "crnn_clip_momentum_step": (c_int, [c_void_p, c_float, c_float, c_float, c_float, c_float, c_void_p]),
    "crnn_clip_rmsprop_step": (c_int, [c_void_p, c_float, c_float, c_float, c_float, c_float, c_float, c_float, c_void_p]),
    "crnn_last_grad_norm": (c_int, [c_void_p, c_float, ctypes.POINTER(c_float), c_void_p]),
    "crnn_model_set_data_parallel": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "crnn_model_set_grad_ready_callback": (c_int, [c_void_p, c_void_p, c_void_p]),
    "crnn_model_set_backward_sm_reserve": (c_int, [c_void_p, c_int]),
    "crnn_peer_inbox_bytes": (c_size_t, []),
    "crnn_peer_inbox_create": (c_int, [ctypes.POINTER(c_void_p), c_void_p]),
    "crnn_peer_inbox_open": (c_int, [c_void_p, ctypes.POINTER(c_void_p)]),
    "crnn_peer_inbox_close": (c_int, [c_void_p]),
    "crnn_peer_inbox_destroy": (c_int, [c_void_p]),
    "crnn_model_set_peers": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "crnn_peer_error": (c_int, [c_void_p, ctypes.POINTER(c_int)]),
    "crnn_test_gemm_tn_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "crnn_test_gemm_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
}

ALLREDUCE_FN = ctypes.CFUNCTYPE(c_int, c_void_p, c_void_p, c_size_t, c_int, c_void_p)
GRAD_READY_FN = ctypes.CFUNCTYPE(None, c_void_p, c_int64, c_int64, c_void_p)

_lib = None


class CrnnError(RuntimeError):
    pass


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CrnnError(f"{LIB_PATH} is missing: run `python build.py` (or __graft_entry__.build()). "
                        "There is no CPU fallback for this path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status):
    if status != 0:
        lib = load()
        raise CrnnError(f"{lib.crnn_status_string(status).decode()}: {lib.crnn_last_error().decode()}")
