"""ctypes binding of libdwm_b200.so (the C ABI declared in include/dwm_b200.h).

There is deliberately no fallback: if the shared library is missing or a call
fails, a RuntimeError is raised.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdwm_b200.so")

DWM_BF16, DWM_F16, DWM_F32, DWM_E4M3 = 0, 1, 2, 3
ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF, ACT_SILU, ACT_RELU, ACT_QUICK_GELU = 0, 1, 2, 3, 4, 5
EPI_STORE, EPI_GEGLU, EPI_QKNORM, EPI_RESID, EPI_F32, EPI_GEGLU_TANH = 0, 1, 2, 3, 4, 5

_i64 = ctypes.c_int64
_p = ctypes.c_void_p


class LinearArgs(ctypes.Structure):
    _fields_ = [
        ("M", _i64), ("N", _i64), ("K", _i64),
        ("A", _p), ("lda", _i64),
        ("W", _p), ("ldw", _i64),
        ("bias", _p),
        ("dtype", ctypes.c_int), ("epilogue", ctypes.c_int),
        ("act", ctypes.c_int),
        ("out", _p), ("ldo", _i64),
        ("rows_per_item", _i64), ("out_item_stride", _i64),
        ("out_row_offset", _i64),
        ("q_norm_weight", _p), ("k_norm_weight", _p), ("qk_region", _i64),
        ("eps", ctypes.c_float), ("qk_norm_regions", ctypes.c_int),
        ("resid", _p), ("ldr", _i64), ("resid_row_mod", _i64),
        ("gate", _p), ("gate_ld", _i64),
        ("blend_x", _p), ("ldx", _i64),
        ("alpha", _p), ("rows_per_batch", _i64),
        ("peer_out", _p * 8), ("n_peer_out", ctypes.c_int),
        ("a_scale", _p), ("w_scale", _p), ("out_dtype", ctypes.c_int),
    ]


class AttentionArgs(ctypes.Structure):
    _fields_ = [
        ("qkv", _p), ("ld", _i64), ("D", _i64),
        ("heads", ctypes.c_int), ("head_dim", ctypes.c_int),
        ("dtype", ctypes.c_int),
        ("group_dims", _i64 * 3), ("group_strides", _i64 * 3),
        ("seq", ctypes.c_int), ("inner", ctypes.c_int),
        ("stride_outer", _i64), ("stride_inner", _i64),
        ("out", _p), ("ldo", _i64),
        ("out_group_strides", _i64 * 3),
        ("out_stride_outer", _i64), ("out_stride_inner", _i64),
        ("split", ctypes.c_int), ("out2", _p), ("ldo2", _i64),
        ("mask", _p), ("mask_div", ctypes.c_int), ("n_outer", ctypes.c_int),
        ("scale", ctypes.c_float),
        ("kv", _p), ("ld_kv", _i64), ("k_col", _i64), ("v_col", _i64),
        ("kv_group_strides", _i64 * 3),
        ("seq_kv", ctypes.c_int), ("inner_kv", ctypes.c_int),
        ("kv_stride_outer", _i64), ("kv_stride_inner", _i64),
        ("mask_q_offset", ctypes.c_int),
    ]


class LayerNormArgs(ctypes.Structure):
    _fields_ = [
        ("M", _i64), ("D", _i64),
        ("x", _p), ("ldx", _i64),
        ("add_item", _p), ("add_item_ld", _i64),
        ("add_full", _p), ("add_full_ld", _i64),
        ("rows_per_item", _i64),
        ("sum_out", _p), ("ld_sum", _i64),
        ("weight", _p), ("bias", _p), ("eps", ctypes.c_float),
        ("shift", _p), ("scale", _p), ("shift2", _p), ("scale2", _p),
        ("mod_ld", _i64),
        ("out", _p), ("ldo", _i64), ("out2", _p), ("ldo2", _i64),
        ("dtype", ctypes.c_int),
        ("out_scale", _p), ("out2_scale", _p),
    ]


class ConvArgs(ctypes.Structure):
    _fields_ = [
        ("x", _p), ("nb", _i64), ("tp", _i64), ("h", _i64), ("w", _i64),
        ("c_in", _i64),
        ("weight", _p), ("kt", ctypes.c_int), ("kh", ctypes.c_int),
        ("kw", ctypes.c_int), ("c_out", _i64),
        ("bias", _p), ("dtype", ctypes.c_int), ("epilogue", ctypes.c_int),
        ("act", ctypes.c_int),
        ("out", _p), ("ldo", _i64), ("resid", _p), ("ldr", _i64),
        ("resid_per_item", ctypes.c_int), ("rows_per_item", _i64),
        ("blend_x", _p), ("ldx", _i64), ("alpha", _p), ("rows_per_batch", _i64),
        ("a_scale", _p), ("w_scale", _p),
    ]


_lib = None

# name -> (restype, argtypes); every symbol include/dwm_b200.h declares.
SYMBOLS = {
    "dwm_b200_version": (ctypes.c_char_p, []),
    "dwm_b200_last_error": (ctypes.c_char_p, []),
    "dwm_b200_set_option": (ctypes.c_int, [ctypes.c_char_p, ctypes.c_int]),
    "dwm_b200_linear": (ctypes.c_int, [ctypes.POINTER(LinearArgs), _p]),
    "dwm_b200_attention": (ctypes.c_int, [ctypes.POINTER(AttentionArgs), _p]),
    "dwm_b200_attention_text": (ctypes.c_int, [ctypes.POINTER(AttentionArgs), ctypes.c_int, _p,
                                               _p]),
    "dwm_b200_layernorm": (ctypes.c_int, [ctypes.POINTER(LayerNormArgs), _p]),
    "dwm_b200_rmsnorm": (ctypes.c_int, [_p, _i64, _i64, _i64, _p, ctypes.c_float, _p, _i64,
                                        ctypes.c_int, _p]),
    "dwm_b200_embed": (ctypes.c_int, [_p, _i64, _i64, _p, _i64, _p, _i64, _p, _i64, _p]),
    "dwm_b200_quantize_rows": (ctypes.c_int, [_p, _i64, _i64, _i64, ctypes.c_int, _p, _i64,
                                              _p, _p]),
    "dwm_b200_act_cast": (ctypes.c_int, [_p, _p, _i64, ctypes.c_int, ctypes.c_int, _p]),
    "dwm_b200_sinusoid": (ctypes.c_int, [_p, _i64, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_float, _p, _i64, ctypes.c_int, _p]),
    "dwm_b200_patchify": (ctypes.c_int, [_p, _i64, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_int, ctypes.c_int, _p, _i64,
                                         ctypes.c_int, _p]),
    "dwm_b200_cfg_euler_step": (ctypes.c_int, [
        _p, _i64, ctypes.c_int, ctypes.c_float, _i64, _i64, _i64, ctypes.c_int,
        ctypes.c_int, ctypes.c_int, ctypes.c_int, _p, _p, ctypes.c_int, _p, _p,
        _p, ctypes.c_int, _p]),
    "dwm_b200_conv": (ctypes.c_int, [ctypes.POINTER(ConvArgs), _p]),
    "dwm_b200_axpy": (ctypes.c_int, [_p, _p, _i64, ctypes.c_float, _p]),
    "dwm_b200_softmax_rows": (ctypes.c_int, [_p, _i64, _i64, _i64, ctypes.c_float, _p, _i64,
                                            ctypes.c_int, _p]),
    "dwm_b200_lincomb2": (ctypes.c_int, [_p, _p, _p, _p, _i64, _i64, _p, _p]),
    "dwm_b200_cfg_dpmpp_step": (ctypes.c_int, [_p, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                               _i64, _p, _p, _p, _p]),
    "dwm_b200_cfg_ddim_step": (ctypes.c_int, [
        _p, ctypes.c_int, ctypes.c_float, _i64, _i64, _p, ctypes.c_int, _p,
        ctypes.c_int, ctypes.c_float, ctypes.c_int, _p, ctypes.c_int, _p]),
    "dwm_b200_groupnorm_stats": (ctypes.c_int, [_p, _i64, _i64, ctypes.c_int,
                                                ctypes.c_int, _p, _p]),
    "dwm_b200_spatialnorm_silu": (ctypes.c_int, [
        _p, _i64, _i64, _i64, _i64, ctypes.c_int, ctypes.c_int, _p, ctypes.c_float,
        _p, _p, _p, _p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _p,
        _i64, _i64, ctypes.c_int, _p]),
    "dwm_b200_groupnorm_silu_e4m3": (ctypes.c_int, [
        _p, _i64, _i64, _i64, _i64, ctypes.c_int, ctypes.c_int, _p, ctypes.c_float,
        _p, _p, ctypes.c_int, _p, _i64, _i64, _p, _p]),
    "dwm_b200_spatialnorm_silu_e4m3": (ctypes.c_int, [
        _p, _i64, _i64, _i64, _i64, ctypes.c_int, ctypes.c_int, _p, ctypes.c_float,
        _p, _p, _p, _p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _p,
        _i64, _i64, _p, _p, _p, ctypes.c_int, _p]),
    "dwm_b200_groupnorm_silu_halo": (ctypes.c_int, [
        _p, _i64, _i64, _i64, _i64, ctypes.c_int, ctypes.c_int, _p, _i64, ctypes.c_float,
        _p, _p, ctypes.c_int, _p, _p, _i64, _p, _i64, ctypes.c_int, _p]),
    "dwm_b200_groupnorm_silu_e4m3_amax": (ctypes.c_int, [
        _p, _i64, _i64, _i64, _i64, ctypes.c_int, ctypes.c_int, _p, _i64, ctypes.c_float,
        _p, _p, ctypes.c_int, _p, _p]),
    "dwm_b200_groupnorm_silu_e4m3_halo": (ctypes.c_int, [
        _p, _i64, _i64, _i64, _i64, ctypes.c_int, ctypes.c_int, _p, _i64, ctypes.c_float,
        _p, _p, ctypes.c_int, _p, _p, _p, _i64, _p, _i64, _p, _p]),
    "dwm_b200_upsample_nearest": (ctypes.c_int, [
        _p, _i64, _i64, _i64, _i64, ctypes.c_int, ctypes.c_int, _p, ctypes.c_int, _p]),
    "dwm_b200_euler_step_by_indices": (ctypes.c_int, [
        _p, _p, _i64, _i64, _p, _p, ctypes.c_int, ctypes.c_int, _p]),
}


def load():
    """Loads the shared library (building nothing). Raises if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "{} not found: run `python -m opendwm_b200.build` (no CPU "
                "fallback exists)".format(LIB_PATH))
        lib = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SYMBOLS.items():
            fn = getattr(lib, name)
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
    return _lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().dwm_b200_last_error().decode("utf-8", "replace")
        raise RuntimeError("{} failed (rc={}): {}".format(what, rc, msg))


def set_option(name: str, value: int):
    check(load().dwm_b200_set_option(name.encode(), int(value)), "dwm_b200_set_option")
