"""ctypes binding of libtensorrec_b200.so (the C ABI declared in include/tensorrec_b200.h).

There is no CPU fallback: if the library cannot be loaded, or no CUDA device is present, every compute call raises.
"""
import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libtensorrec_b200.so')

TRK_OK = 0
TRK_ERR_ARG = -1
TRK_ERR_CUDA = -2
TRK_ERR_UNSUPPORTED = -3


class TrkUnsupportedError(RuntimeError):
    """The shape is outside what the fused tensor-core kernel supports (callers may pick another kernel)."""


_c_i32, _c_i64, _c_p, _c_sz = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p, ctypes.c_size_t

# name -> (restype, argtypes); mirrors include/tensorrec_b200.h one to one
SIGNATURES = {
    'trk_version': (ctypes.c_int, []),
    'trk_last_error': (ctypes.c_char_p, []),
    'trk_csr_gather_reduce_f32': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_i64, _c_i32, _c_i32, _c_i32, _c_p, _c_p,
                                                 _c_i32, _c_p, _c_p, _c_p, _c_p]),
    'trk_split_f32_to_f16x2': (ctypes.c_int, [_c_p, _c_i64, _c_i32, _c_i32, _c_p, _c_i32, _c_p, _c_p]),
    'trk_l2_normalize_rows_f32': (ctypes.c_int, [_c_p, _c_i64, _c_i32, _c_p]),
    'trk_csr_project_biases_f32': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_i64, _c_p, _c_p]),
    'trk_score_f32': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32, _c_i32, _c_p]),
    'trk_score_attention_f32': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32,
                                               _c_p]),
    'trk_rank_full_workspace_bytes': (_c_sz, [_c_i64, _c_i64]),
    'trk_rank_full': (ctypes.c_int, [_c_p, _c_p, _c_i64, _c_i64, _c_p, _c_sz, _c_p]),
    'trk_order_from_ranks': (ctypes.c_int, [_c_p, _c_i64, _c_p, _c_p]),
    'trk_score_topk_max_k': (ctypes.c_int, [_c_i32]),
    'trk_pack_item_meta': (ctypes.c_int, [_c_p, _c_p, _c_i64, _c_p, _c_i64, _c_p]),
    'trk_score_topk_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32, _c_i32,
                                            _c_i32, _c_p, _c_p, _c_p, _c_p]),
    'trk_score_topk_f16x3_excl': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32, _c_i32,
                                                 _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p]),
    'trk_exclusion_positions': (ctypes.c_int, [_c_p, _c_i64, _c_p, _c_p, _c_p, _c_i64, _c_p, _c_p]),
    'trk_score_dense_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_p, _c_i64,
                                             _c_p]),
    'trk_score_dense_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_p, _c_i64,
                                                    _c_p, _c_p, _c_p]),
    'trk_score_topk_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32, _c_i32,
                                                   _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p]),
    'trk_score_dense_tastes_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_i64,
                                                    _c_i32, _c_p, _c_i64, _c_p]),
    'trk_score_topk_tastes_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_i64, _c_i32,
                                                   _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p]),
    'trk_score_topk_wide_list_capacity': (ctypes.c_int, [_c_i32]),
    'trk_score_topk_wide_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32,
                                                        _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p,
                                                        _c_p, _c_p]),
    'trk_score_topk_wide_tastes_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_i64,
                                                        _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p,
                                                        _c_p, _c_p]),
    'trk_score_count_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32, _c_i32,
                                             _c_p, _c_p, _c_p, _c_p, _c_p, _c_i32, _c_p, _c_p, _c_p, _c_p]),
    'trk_score_count_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32,
                                                    _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i32, _c_p, _c_p, _c_p,
                                                    _c_p, _c_p, _c_p]),
    'trk_score_count_tastes_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_i64,
                                                    _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i32, _c_p,
                                                    _c_p, _c_p, _c_p]),
    'trk_score_dense_tastes_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_i64,
                                                           _c_i32, _c_p, _c_i64, _c_p, _c_p, _c_p]),
    'trk_score_topk_tastes_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_i64,
                                                          _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p,
                                                          _c_p, _c_p, _c_p]),
    'trk_score_topk_wide_tastes_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64,
                                                               _c_i64, _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p,
                                                               _c_p, _c_p, _c_p, _c_p, _c_p, _c_p]),
    'trk_score_count_tastes_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_i64,
                                                           _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i32,
                                                           _c_p, _c_p, _c_p, _c_p, _c_p, _c_p]),
    'trk_score_pairs_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_p, _c_p, _c_p,
                                             _c_p, _c_i32, _c_p, _c_i32, _c_p]),
    'trk_score_pairs_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_p, _c_p,
                                                    _c_p, _c_p, _c_i32, _c_p, _c_i32, _c_p, _c_p, _c_p]),
    'trk_score_pairs_tastes_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_i64,
                                                    _c_i32, _c_p, _c_p, _c_p, _c_p, _c_i32, _c_p, _c_i32, _c_p]),
    'trk_score_pairs_tastes_euclid_f16x3': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_i64,
                                                           _c_i32, _c_p, _c_p, _c_p, _c_p, _c_i32, _c_p, _c_i32, _c_p,
                                                           _c_p, _c_p]),
    'trk_select_topk_lists': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i64, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_i64,
                                             _c_p]),
    'trk_topk_merge': (ctypes.c_int, [_c_p, _c_p, _c_i64, _c_i32, _c_i32, _c_i32, _c_i64, _c_i64, _c_p, _c_p, _c_i64,
                                      _c_p, _c_i32, _c_p]),
    'trk_topk_merge_dedup_pair': (ctypes.c_int, [_c_p, _c_p, _c_i64, _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_p, _c_p,
                                                 _c_i64, _c_p]),
    'trk_score_filter_max_k': (ctypes.c_int, []),
    'trk_score_filter_list_width': (ctypes.c_int, []),
    'trk_operand_stats': (ctypes.c_int, [_c_p, _c_p, _c_i64, _c_i32, _c_p, _c_p, _c_p]),
    'trk_rescale_hi_global': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_i64, _c_i32, _c_p, _c_p]),
    'trk_pack_item_bias': (ctypes.c_int, [_c_p, _c_p, _c_i64, _c_p, _c_i64, _c_p, _c_p, _c_p, _c_p]),
    'trk_score_filter_f16': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64,
                                            _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p]),
    'trk_score_filter_f16_excl': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i64,
                                                 _c_i64, _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p,
                                                 _c_p]),
    'trk_rescore_topk_split': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64,
                                              _c_i32, _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_i64, _c_p, _c_p]),
    'trk_select_flagged_rows': (ctypes.c_int, [_c_p, _c_i64, _c_p, _c_i32, _c_p, _c_p]),
    'trk_gather_operand_rows': (ctypes.c_int, [_c_p, _c_p, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_i32, _c_p, _c_p, _c_p,
                                               _c_p]),
    'trk_scatter_topk_rows': (ctypes.c_int, [_c_p, _c_p, _c_i32, _c_p, _c_p, _c_i64, _c_i32, _c_p, _c_p, _c_i64, _c_p]),
    'trk_operand_half_sqnorm': (ctypes.c_int, [_c_p, _c_p, _c_i64, _c_i32, _c_p, _c_p]),
    'trk_topk_euclidean_finish': (ctypes.c_int, [_c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_p]),
    'trk_score_wide_max_k': (ctypes.c_int, []),
    'trk_score_wide_list_capacity': (ctypes.c_int, [_c_i32]),
    'trk_score_wide_f16': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32,
                                          _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p]),
    'trk_score_wide_f16_excl': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64,
                                               _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p]),
    'trk_select_wide_topk': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i32, _c_i32, _c_p, _c_p,
                                            _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p,
                                            _c_i64, _c_p, _c_p]),
    'trk_sample_items': (ctypes.c_int, [_c_i64, _c_i64, _c_i32, _c_i32, ctypes.c_uint64, ctypes.c_uint32, _c_p, _c_p]),
    'trk_sample_stream_u64': (ctypes.c_uint64, [ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32]),
    'trk_wmrb_step': (ctypes.c_int, [_c_p, _c_p, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_i64, _c_i64, _c_i32,
                                     _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p]),
    'trk_wmrb_step_tastes': (ctypes.c_int, [_c_p, _c_p, _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p,
                                            _c_p, _c_p, _c_i64, _c_i64, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p, _c_p,
                                            _c_p, _c_p, _c_p]),
    'trk_serial_loss_workspace_bytes': (_c_sz, [_c_i64]),
    'trk_serial_loss_step': (ctypes.c_int, [_c_i32, _c_p, _c_p, _c_i32, _c_i32, _c_i32, _c_i32, _c_p, _c_p, _c_p, _c_p,
                                            _c_p, _c_i64, _c_i64, _c_i32, _c_i64, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p, _c_p,
                                            _c_sz, _c_p]),
    'trk_l2_normalize_rows_step_f32': (ctypes.c_int, [_c_p, _c_i64, _c_i32, _c_i32, _c_p, _c_p, _c_p]),
    'trk_f32_to_bf16': (ctypes.c_int, [_c_p, _c_i64, _c_p, _c_p]),
    'trk_adam_step_f32': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_i64, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                         ctypes.c_float, ctypes.c_float, _c_p]),
    'trk_relu_layer_workspace_bytes': (_c_sz, [_c_i64, _c_i32, _c_i32]),
    'trk_relu_layer_forward_f32': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_i64, _c_i32, _c_i32, _c_p, _c_p]),
    'trk_relu_layer_backward_f32': (ctypes.c_int, [_c_p, _c_p, _c_p, _c_p, _c_i64, _c_i32, _c_i32, _c_p, _c_p, _c_p,
                                                   _c_sz, _c_p]),
}

_lib = None
_lock = threading.Lock()


def load(build_if_missing=True):
    """Loads (building first if the .so is absent and nvcc is available) and returns the ctypes library."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            if not build_if_missing:
                raise RuntimeError('tensorrec_b200: %s is missing; run `python -m tensorrec_b200.csrc.build`' % LIB_PATH)
            from .csrc.build import build
            build()
        lib = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)          # AttributeError here == the library does not export the ABI
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
        return _lib


def last_error():
    return load().trk_last_error().decode('utf-8', 'replace')


launch_count = 0   # successful kernel-launching ABI calls so far (bench.py reports the delta over its timed region)


def check(rc, what):
    global launch_count
    if rc == TRK_OK:
        launch_count += 1
        return
    msg = '%s: %s' % (what, last_error())
    if rc == TRK_ERR_ARG:
        raise ValueError(msg)
    if rc == TRK_ERR_UNSUPPORTED:
        raise TrkUnsupportedError(msg)
    raise RuntimeError(msg)
