"""ctypes binding of librten_b200.so (the C ABI in include/rten_b200.h).

The library is the product; this module only marshals descriptors.  It fails loudly when the
shared object is missing or no H100 is present -- there is no CPU fallback."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "librten_b200.so")

RTEN_MAX_DIMS = 8
RTEN_DEVICE_HOST = -1
RTEN_F32, RTEN_I32, RTEN_I8, RTEN_U8 = 0, 1, 2, 3

STATUS_NAMES = {
    0: "Ok", 1: "CastFailed", 2: "UnsupportedType", 3: "IncompatibleInputShapes", 4: "MissingInputs",
    5: "InvalidValue", 6: "UnsupportedValue", 7: "UnsupportedOutput", 100: "Cuda", 101: "Nccl",
}


class RtenTensor(C.Structure):
    _fields_ = [
        ("data", C.c_void_p),
        ("dtype", C.c_int32),
        ("ndim", C.c_int32),
        ("shape", C.c_int64 * RTEN_MAX_DIMS),
        ("strides", C.c_int64 * RTEN_MAX_DIMS),
        ("device", C.c_int32),
        ("_reserved", C.c_int32),
    ]


class RtenModelInputOpts(C.Structure):
    _fields_ = [("writable", C.c_int32), ("grow_axis", C.c_int32), ("capacity", C.c_int64)]


class RtenConvParams(C.Structure):
    _fields_ = [
        ("pads", C.c_int32 * 4),
        ("auto_pad_same", C.c_int32),
        ("groups", C.c_int32),
        ("strides", C.c_int32 * 2),
        ("dilations", C.c_int32 * 2),
        ("n_strides", C.c_int32),
        ("n_dilations", C.c_int32),
    ]


class RtenConvTransposeParams(C.Structure):
    _fields_ = [
        ("pads", C.c_int32 * 4),
        ("auto_pad_same", C.c_int32),
        ("groups", C.c_int32),
        ("strides", C.c_int32 * 2),
        ("dilations", C.c_int32 * 2),
        ("output_padding", C.c_int32 * 2),
        ("n_pads", C.c_int32),
        ("n_strides", C.c_int32),
        ("n_dilations", C.c_int32),
        ("n_output_padding", C.c_int32),
    ]


class RtenAttentionParams(C.Structure):
    _fields_ = [("is_causal", C.c_int32), ("q_num_heads", C.c_int32), ("kv_num_heads", C.c_int32), ("scale", C.c_float),
                ("softcap", C.c_float)]


class RtenGqaParams(C.Structure):
    _fields_ = [("num_heads", C.c_int32), ("kv_num_heads", C.c_int32), ("scale", C.c_float), ("do_rotary", C.c_int32),
                ("rotary_interleaved", C.c_int32), ("local_window_size", C.c_int32), ("softcap", C.c_float)]


class RtenMhaParams(C.Structure):
    _fields_ = [("num_heads", C.c_int32), ("scale", C.c_float), ("mask_filter_value", C.c_float), ("unidirectional", C.c_int32)]


class RtenActivation(C.Structure):
    _fields_ = [("kind", C.c_int32), ("alpha", C.c_float), ("beta", C.c_float)]


class RtenResizeParams(C.Structure):
    _fields_ = [("mode", C.c_int32), ("coord_mode", C.c_int32), ("nearest_mode", C.c_int32), ("n", C.c_int32),
                ("scales", C.c_float * 4), ("sizes", C.c_int64 * 4), ("use_sizes", C.c_int32)]


class RtenRnnParams(C.Structure):
    _fields_ = [("direction", C.c_int32), ("hidden_size", C.c_int32), ("linear_before_reset", C.c_int32)]


_TP = C.POINTER(RtenTensor)
_vp = C.c_void_p

_SIGNATURES = {
    "rten_b200_version": (C.c_char_p, []),
    "rten_b200_ctx_create": (C.c_int, [C.c_int, _vp, C.c_size_t, C.POINTER(_vp)]),
    "rten_b200_ctx_destroy": (None, [_vp]),
    "rten_b200_last_error": (C.c_char_p, [_vp]),
    "rten_b200_sync": (C.c_int, [_vp]),
    "rten_b200_set_f32_mode": (C.c_int, [_vp, C.c_int]),
    "rten_b200_set_autotune": (C.c_int, [_vp, C.c_int]),
    "rten_b200_save_plans": (C.c_int, [_vp, C.c_char_p]),
    "rten_b200_load_plans": (C.c_int, [_vp, C.c_char_p]),
    "rten_b200_alloc": (C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    "rten_b200_free": (C.c_int, [_vp, _vp]),
    "rten_b200_host_alloc": (C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    "rten_b200_host_free": (C.c_int, [_vp, _vp]),
    "rten_b200_copy": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_launch_count": (C.c_uint64, [_vp]),
    "rten_b200_debug_forced_plans": (C.c_int, [_vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "rten_b200_graph_begin": (C.c_int, [_vp]),
    "rten_b200_graph_end": (C.c_int, [_vp, C.POINTER(_vp)]),
    "rten_b200_graph_launch": (C.c_int, [_vp, _vp]),
    "rten_b200_graph_destroy": (None, [_vp]),
    "rten_b200_prepack_b": (C.c_int, [_vp, _TP, C.POINTER(_vp)]),
    "rten_b200_prepack_conv_weight": (C.c_int, [_vp, _TP, C.c_int, C.POINTER(_vp)]),
    "rten_b200_packed_free": (None, [_vp, _vp]),
    "rten_b200_gemm": (C.c_int, [_vp, _TP, _TP, _TP, C.c_float, C.c_float, C.c_int, C.c_int, _TP]),
    "rten_b200_matmul": (C.c_int, [_vp, _TP, _TP, _vp, _TP, C.c_float, _TP]),
    "rten_b200_matmul_ex": (C.c_int, [_vp, _TP, _TP, _vp, _TP, C.c_float, _TP, C.c_int, _TP]),
    "rten_b200_matmul_integer": (C.c_int, [_vp, _TP, _TP, _vp, _TP, _TP, _TP, _TP]),
    "rten_b200_matmul_integer_ex": (C.c_int, [_vp, _TP, _TP, _vp, _TP, _TP, _TP, _TP, _TP, _TP, C.c_int, _TP, _TP]),
    "rten_b200_matmul_nbits": (C.c_int, [_vp, _TP, _TP, _TP, C.c_int, C.c_int, _TP]),
    "rten_b200_conv2d": (C.c_int, [_vp, _TP, _TP, _vp, _TP, C.POINTER(RtenConvParams), _TP]),
    "rten_b200_conv2d_ex": (C.c_int, [_vp, _TP, _TP, _vp, _TP, C.POINTER(RtenConvParams), _TP, C.c_int, _TP]),
    "rten_b200_conv2d_act": (C.c_int, [_vp, _TP, _TP, _vp, _TP, C.POINTER(RtenConvParams), _TP, C.POINTER(RtenActivation), _TP]),
    "rten_b200_conv2d_projected": (C.c_int, [_vp, _TP, _TP, _vp, _TP, C.POINTER(RtenConvParams), _TP, _TP, _vp, _TP,
                                             C.POINTER(RtenConvParams), C.c_int, _TP]),
    "rten_b200_conv2d_chained": (C.c_int, [_vp, _TP, _TP, _vp, _TP, C.POINTER(RtenConvParams), _TP, _TP, _TP, _vp, _TP,
                                           C.POINTER(RtenConvParams), C.c_int, _TP, _vp, _TP, C.POINTER(RtenConvParams),
                                           C.c_int, _TP, _TP]),
    "rten_b200_conv_transpose": (C.c_int, [_vp, _TP, _TP, _vp, _TP, C.POINTER(RtenConvTransposeParams), _TP]),
    "rten_b200_prepack_conv_transpose_weight": (C.c_int, [_vp, _TP, C.POINTER(RtenConvTransposeParams), C.POINTER(_vp)]),
    "rten_b200_conv_integer": (C.c_int, [_vp, _TP, _TP, _vp, _TP, _TP, _TP, C.POINTER(RtenConvParams), _TP]),
    "rten_b200_quantized_linear": (C.c_int, [_vp, _TP, _TP, _TP, C.c_float, _TP, _vp, _TP, _TP, _TP, _TP, C.c_int, _TP]),
    "rten_b200_attention": (C.c_int, [_vp, _TP, _TP, _TP, _TP, _TP, C.POINTER(RtenAttentionParams), _TP, _TP, _TP]),
    "rten_b200_rotary_embedding": (C.c_int, [_vp, _TP, _TP, _TP, _TP, C.c_int, C.c_int, C.c_int, _TP]),
    "rten_b200_group_query_attention": (C.c_int, [_vp, _TP, _TP, _TP, _TP, _TP, _TP, _TP, _TP, _TP, _TP, _TP,
                                                  C.POINTER(RtenGqaParams), _TP, _TP, _TP]),
    "rten_b200_multi_head_attention": (C.c_int, [_vp, _TP, _TP, _TP, _TP, _TP, _TP, _TP, _TP, _TP, _TP,
                                                 C.POINTER(RtenMhaParams), _TP, _TP, _TP]),
    "rten_b200_gru": (C.c_int, [_vp, _TP, _TP, _vp, _TP, _TP, _TP, _TP, C.POINTER(RtenRnnParams), _TP, _TP]),
    "rten_b200_lstm": (C.c_int, [_vp, _TP, _TP, _vp, _TP, _TP, _TP, _TP, _TP, _TP, C.POINTER(RtenRnnParams), _TP, _TP, _TP]),
    "rten_b200_softmax": (C.c_int, [_vp, _TP, _TP, C.c_int, C.c_int, _TP]),
    "rten_b200_layer_norm": (C.c_int, [_vp, _TP, _TP, _TP, C.c_int, C.c_float, _TP]),
    "rten_b200_rms_norm": (C.c_int, [_vp, _TP, _TP, C.c_int, C.c_float, _TP]),
    "rten_b200_skip_layer_norm": (C.c_int, [_vp, _TP, _TP, _TP, _TP, _TP, C.c_float, C.c_int, _TP, _TP]),
    "rten_b200_instance_norm": (C.c_int, [_vp, _TP, _TP, _TP, C.c_float, _TP]),
    "rten_b200_group_norm": (C.c_int, [_vp, _TP, C.c_int, _TP, _TP, _TP, _TP, C.c_float, C.POINTER(RtenActivation), _TP]),
    "rten_b200_batch_norm": (C.c_int, [_vp, _TP, _TP, _TP, _TP, _TP, C.c_float, C.POINTER(RtenActivation), _TP]),
    "rten_b200_erf": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_gelu": (C.c_int, [_vp, _TP, C.c_int, _TP]),
    "rten_b200_dynamic_quantize_linear": (C.c_int, [_vp, _TP, _TP, _TP, _TP, _vp]),
    "rten_b200_comm_unique_id": (C.c_int, [_vp]),
    "rten_b200_comm_create": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.POINTER(_vp)]),
    "rten_b200_comm_destroy": (None, [_vp]),
    "rten_b200_comm_uses_peer_memory": (C.c_int, [_vp]),
    "rten_b200_comm_timeouts": (C.c_int, [_vp]),
    "rten_b200_relu": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_sigmoid": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_silu": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_hard_sigmoid": (C.c_int, [_vp, _TP, C.c_float, C.c_float, _TP]),
    "rten_b200_hard_swish": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_clip": (C.c_int, [_vp, _TP, _TP, _TP, _TP]),
    "rten_b200_add": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_mul": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_sub": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_div": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_pow": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_sqrt": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_reciprocal": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_exp": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_tanh": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_neg": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_abs": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_where": (C.c_int, [_vp, _TP, _TP, _TP, _TP]),
    "rten_b200_equal": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_less": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_less_or_equal": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_greater": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_greater_or_equal": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_and": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_or": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_xor": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_not": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_trilu": (C.c_int, [_vp, _TP, C.c_int64, C.c_int, _TP]),
    "rten_b200_expand": (C.c_int, [_vp, _TP, C.POINTER(C.c_int64), C.c_int, _TP]),
    "rten_b200_slice": (C.c_int, [_vp, _TP, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                  C.c_int, _TP]),
    "rten_b200_split": (C.c_int, [_vp, _TP, C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_int, _TP, C.c_int, C.POINTER(C.c_int32)]),
    "rten_b200_reduce_sum": (C.c_int, [_vp, _TP, C.POINTER(C.c_int32), C.c_int, C.c_int, _TP]),
    "rten_b200_reduce_mean": (C.c_int, [_vp, _TP, C.POINTER(C.c_int32), C.c_int, C.c_int, _TP]),
    "rten_b200_topk": (C.c_int, [_vp, _TP, C.c_int64, C.c_int, C.c_int, C.c_int, _TP, _TP]),
    "rten_b200_arg_max": (C.c_int, [_vp, _TP, C.c_int, C.c_int, _TP]),
    "rten_b200_arg_min": (C.c_int, [_vp, _TP, C.c_int, C.c_int, _TP]),
    "rten_b200_conv_integer_ex": (C.c_int, [_vp, _TP, _TP, _vp, _TP, _TP, _TP, _TP, C.POINTER(RtenConvParams), _TP, _TP, C.c_int, _TP, _TP]),
    "rten_b200_range_reset": (C.c_int, [_vp, _TP]),
    "rten_b200_dynamic_quantize_linear_ranged": (C.c_int, [_vp, _TP, _TP, _TP, _TP, _TP, _vp]),
    "rten_b200_max_pool": (C.c_int, [_vp, _TP, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), _TP]),
    "rten_b200_global_average_pool": (C.c_int, [_vp, _TP, _TP]),
    "rten_b200_average_pool": (C.c_int, [_vp, _TP, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int, _TP]),
    "rten_b200_resize": (C.c_int, [_vp, _TP, C.POINTER(RtenResizeParams), _TP]),
    "rten_b200_concat": (C.c_int, [_vp, C.POINTER(_TP), C.c_int, C.c_int, _TP]),
    "rten_b200_gather_rows": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_scatter_rows": (C.c_int, [_vp, _TP, _TP, _TP]),
    "rten_b200_model_load": (C.c_int, [_vp, _vp, C.c_size_t, C.POINTER(_vp)]),
    "rten_b200_model_free": (None, [_vp]),
    "rten_b200_model_num_inputs": (C.c_int32, [_vp]),
    "rten_b200_model_num_outputs": (C.c_int32, [_vp]),
    "rten_b200_model_input_name": (C.c_char_p, [_vp, C.c_int32]),
    "rten_b200_model_output_name": (C.c_char_p, [_vp, C.c_int32]),
    "rten_b200_model_num_nodes": (C.c_int32, [_vp]),
    "rten_b200_model_node_op": (C.c_char_p, [_vp, C.c_int32]),
    "rten_b200_model_summary": (C.c_char_p, [_vp]),
    "rten_b200_model_run": (C.c_int, [_vp, C.c_int32, C.POINTER(C.c_char_p), _TP, C.c_int32, C.POINTER(C.c_char_p), _TP]),
    "rten_b200_model_run_ex": (C.c_int, [_vp, C.c_int32, C.POINTER(C.c_char_p), _TP, C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), _TP,
                                         C.POINTER(C.c_int32)]),
    "rten_b200_onnx_summary": (C.c_int, [_vp, C.c_size_t, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]),
}

_lib = None


def declared_symbols():
    return sorted(_SIGNATURES)


def load():
    """Load the CUDA library.  Raises if it has not been built -- never falls back to anything."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(rten_b200 has no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib
