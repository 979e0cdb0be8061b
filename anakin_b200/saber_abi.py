"""ctypes declaration of the C ABI in include/b200_saber.h (libb200saber.so).

This is the thin Python host mirror used by the tests, bench.py and the Python
`Net` front end; it adds no arithmetic of its own.  There is NO CPU fallback: if the
library is missing `load()` raises, and on a machine without an sm_90 (H100) GPU every
compute entry point returns SaberWrongDevice (255).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# ANAKIN_B200_LIBDIR: alternative directory holding both .so files (A/B experiments between builds)
_LIBDIR = os.environ.get("ANAKIN_B200_LIBDIR") or os.path.join(_HERE, "lib")
LIB_PATH = os.path.join(_LIBDIR, "libb200saber.so")

# SaberStatus (reference saber/saber_types.h:223-233)
SUCCESS = -1
NOT_INITIALIZED, INVALID_VALUE, UNIMPL_ERROR, WRONG_DEVICE = 1, 3, 127, 255
# DataType (reference saber/saber_types.h:205-222)
HALF, FLOAT, INT8, INT32, UINT8 = 0, 1, 3, 5, 7
POOL_MAX, POOL_AVG_INC, POOL_AVG_EXC = 1, 2, 3
ELT_PROD, ELT_SUM, ELT_MAX = 1, 2, 3
ACT_SIGMOID, ACT_RELU, ACT_TANH, ACT_CLIPPED_RELU, ACT_ELU = 1, 2, 3, 4, 5
MATH_I8, MATH_F16, MATH_TF32, MATH_TF32X3 = 0, 1, 2, 3


class ConvDesc(C.Structure):
    _fields_ = [
        ("math", C.c_int32), ("in_dtype", C.c_int32), ("out_dtype", C.c_int32), ("res_dtype", C.c_int32),
        ("n", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32), ("k", C.c_int32),
        ("ldc", C.c_int32), ("r", C.c_int32), ("s", C.c_int32),
        ("pad_h", C.c_int32), ("pad_w", C.c_int32), ("stride_h", C.c_int32), ("stride_w", C.c_int32),
        ("dil_h", C.c_int32), ("dil_w", C.c_int32), ("relu", C.c_int32), ("neg_slope", C.c_float),
        ("sum_scale", C.c_float), ("fuse_pool", C.c_int32), ("pool_stride", C.c_int32), ("pool_pad", C.c_int32),
        ("pool_floor_as_conv", C.c_int32),
    ]


class PoolDesc(C.Structure):
    _fields_ = [
        ("dtype", C.c_int32), ("type", C.c_int32), ("n", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
        ("c", C.c_int32), ("window_h", C.c_int32), ("window_w", C.c_int32), ("pad_h", C.c_int32),
        ("pad_w", C.c_int32), ("stride_h", C.c_int32), ("stride_w", C.c_int32),
        ("global_pooling", C.c_int32), ("floor_as_conv", C.c_int32), ("reserved", C.c_int32 * 2),
    ]


class StemDesc(C.Structure):
    _fields_ = [
        ("math", C.c_int32), ("out_dtype", C.c_int32), ("n", C.c_int32), ("c", C.c_int32), ("h", C.c_int32),
        ("w", C.c_int32), ("k", C.c_int32), ("ldc", C.c_int32), ("r", C.c_int32), ("s", C.c_int32),
        ("stride_h", C.c_int32), ("stride_w", C.c_int32), ("pad_h", C.c_int32), ("pad_w", C.c_int32),
        ("relu", C.c_int32), ("neg_slope", C.c_float), ("in_inv_scale", C.c_float), ("fuse_pool", C.c_int32),
        ("pool_type", C.c_int32), ("pool_window_h", C.c_int32), ("pool_window_w", C.c_int32),
        ("pool_pad_h", C.c_int32), ("pool_pad_w", C.c_int32), ("pool_stride_h", C.c_int32),
        ("pool_stride_w", C.c_int32), ("pool_global", C.c_int32), ("pool_floor_as_conv", C.c_int32),
        ("monotone_epilogue", C.c_int32), ("reserved", C.c_int32 * 1),
    ]


class FcStreamDesc(C.Structure):
    _fields_ = [
        ("math", C.c_int32), ("in_dtype", C.c_int32), ("out_dtype", C.c_int32),
        ("m", C.c_int32), ("k", C.c_int32), ("ldx", C.c_int32), ("n_out", C.c_int32), ("ldo", C.c_int32),
        ("relu", C.c_int32), ("neg_slope", C.c_float),
    ]


class HeadDesc(C.Structure):
    _fields_ = [("fc", FcStreamDesc), ("hw", C.c_int32), ("pool_max", C.c_int32), ("ldp", C.c_int32)]


# every symbol include/b200_saber.h declares: name -> (restype, argtypes)
_vp, _i, _f, _sz = C.c_void_p, C.c_int32, C.c_float, C.c_size_t
SYMBOLS = {
    "b200_status_string": (C.c_char_p, [C.c_int]),
    "b200_abi_version": (C.c_int, []),
    "b200_device_ok": (C.c_int, [C.c_int]),
    "b200_conv_out_hw": (C.c_int, [C.POINTER(ConvDesc), C.POINTER(_i), C.POINTER(_i)]),
    "b200_conv_pooled_hw": (C.c_int, [C.POINTER(ConvDesc), C.POINTER(_i), C.POINTER(_i)]),
    "b200_conv_packed_weight_bytes": (_sz, [C.POINTER(ConvDesc)]),
    "b200_conv_pack_weights": (C.c_int, [C.POINTER(ConvDesc), _vp, _i, _vp]),
    "b200_conv_plan_create": (C.c_int, [C.POINTER(ConvDesc), _vp, _vp, _vp, C.POINTER(_vp)]),
    "b200_conv_plan_run": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "b200_conv_plan_destroy": (None, [_vp]),
    "b200_conv_plan_info": (C.c_int, [_vp] + [C.POINTER(_i)] * 5),
    "b200_conv_plan_split": (C.c_int, [_vp]),
    "b200_conv_plan_is_slab": (C.c_int, [_vp]),
    "b200_conv_plan_is_persistent": (C.c_int, [_vp]),
    "b200_fc_stream_max_rows": (C.c_int, []),
    "b200_fc_stream_run": (C.c_int, [C.POINTER(FcStreamDesc), _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_head_workspace_bytes": (_sz, [C.POINTER(HeadDesc)]),
    "b200_head_run": (C.c_int, [C.POINTER(HeadDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_dwconv_run": (C.c_int, [C.POINTER(ConvDesc), _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_fc_desc": (C.c_int, [C.POINTER(ConvDesc), _i, _i, _i, _i, _i, _i]),
    "b200_pool_out_hw": (C.c_int, [C.POINTER(PoolDesc), C.POINTER(_i), C.POINTER(_i)]),
    "b200_pool_run": (C.c_int, [C.POINTER(PoolDesc), _vp, _vp, _vp]),
    "b200_softmax_run": (C.c_int, [_vp, _vp, _i, _i, _i, _vp]),
    "b200_softmax_rows": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "b200_eltwise_run": (C.c_int, [_i, _i, _i, _i, _vp, _vp, _vp, _sz, _f, _f, _i, _vp]),
    "b200_activation_run": (C.c_int, [_i, _i, _vp, _vp, _sz, _f, _f, _vp]),
    "b200_scale_run": (C.c_int, [_i, _vp, _vp, _sz, _i, _vp, _vp, _vp]),
    "b200_nchw_to_nhwc": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _i, _i, _f, _i, _vp]),
    "b200_stem_pack": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_nhwc_to_nchw": (C.c_int, [_vp, _i, _vp, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_stem_conv_out_hw": (C.c_int, [C.POINTER(StemDesc), C.POINTER(_i), C.POINTER(_i)]),
    "b200_stem_packed_weight_bytes": (_sz, [C.POINTER(StemDesc)]),
    "b200_stem_pack_weights": (C.c_int, [C.POINTER(StemDesc), _vp, _vp]),
    "b200_stem_conv_info": (C.c_int, [C.POINTER(StemDesc)] + [C.POINTER(_i)] * 5),
    "b200_stem_conv_run": (C.c_int, [C.POINTER(StemDesc), _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_launch_count": (C.c_uint64, []),
}

_lib = None


def load():
    """Load libb200saber.so and bind every declared symbol. Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libb200saber.so is not built (%s). Run `python -m anakin_b200.build` "
            "(or __graft_entry__.build()); there is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    if lib.b200_abi_version() != 1:
        raise RuntimeError("b200_saber ABI version mismatch")
    _lib = lib
    return lib


class SaberError(RuntimeError):
    pass


def check(status, what=""):
    """SABER_CHECK (reference saber/core/common.h:36-40): abort on anything but SaberSuccess."""
    if status != SUCCESS:
        raise SaberError("%s failed: %s (%d)" % (what or "b200 call", load().b200_status_string(status).decode(), status))


def status_string(status):
    return load().b200_status_string(status).decode()
