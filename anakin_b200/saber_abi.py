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
FP8E4M3 = 32          # OCP e4m3fn codes; no reference DataType
POOL_MAX, POOL_AVG_INC, POOL_AVG_EXC = 1, 2, 3
ELT_PROD, ELT_SUM, ELT_MAX = 1, 2, 3
ACT_SIGMOID, ACT_RELU, ACT_TANH, ACT_CLIPPED_RELU, ACT_ELU = 1, 2, 3, 4, 5
MATH_I8, MATH_F16, MATH_TF32X3, MATH_E4M3 = 0, 1, 3, 4
MATH_TF32 = 2         # retired single-pass tf32 kind (ABI version 1): every entry point refuses it as unimplemented
CONV_KERNEL_TILE, CONV_KERNEL_PERSISTENT, CONV_KERNEL_SLAB = 0, 1, 2
IMAGE_INTERLEAVED, IMAGE_YUV_NV12, IMAGE_YUV_I420 = 0, 1, 2
IMAGE_RESIZE_REFERENCE, IMAGE_RESIZE_PIL, IMAGE_RESIZE_PIL_BICUBIC, IMAGE_RESIZE_CV2_LINEAR = 0, 1, 3, 5


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


class ConvPlanChoice(C.Structure):
    """b200_conv_plan_choice_t: the plan b200_conv_plan_choose picks (kernel: CONV_KERNEL_*)."""
    _fields_ = [(f, C.c_int32) for f in ("kernel", "block_n", "split", "stages", "smem_bytes", "grid_x", "grid_y",
                                         "k_steps", "ctas", "tile_h", "tile_w")]


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


class ImageDesc(C.Structure):
    """b200_image_desc_t: network channel i = (image channel src_channel[i] - mean[i]) * scale[i], fp32, no FMA."""
    _fields_ = [("src_channel", C.c_int32 * 4), ("mean", C.c_float * 4), ("scale", C.c_float * 4)]


def image_desc(mean, scale, src_channel=None):
    """ImageDesc for c = len(mean) channels (src_channel defaults to the identity)."""
    c = len(mean)
    src = list(range(c)) if src_channel is None else list(src_channel)
    d = ImageDesc()
    for i in range(min(c, 4)):
        d.src_channel[i], d.mean[i], d.scale[i] = int(src[i]), float(mean[i]), float(scale[i])
    return d


class ImageResizeDesc(C.Structure):
    """b200_image_resize_desc_t: n images of c channels resized and cropped to out_h x out_w."""
    _fields_ = [("n", C.c_int32), ("c", C.c_int32), ("out_h", C.c_int32), ("out_w", C.c_int32)]


class ImageResizeEntry(C.Structure):
    """b200_image_resize_entry_t: one image of the device table (byte offset, source, resized and crop geometry)."""
    _fields_ = [("offset", C.c_int64), ("h", C.c_int32), ("w", C.c_int32), ("rh", C.c_int32), ("rw", C.c_int32),
                ("top", C.c_int32), ("left", C.c_int32)]


class ImageCropEntry(C.Structure):
    """b200_image_crop_entry_t: one box of the crop table (r: the frame's offset, the box's size and geometry; then the
    frame's size and the box's origin in it)."""
    _fields_ = [("r", ImageResizeEntry), ("frame_h", C.c_int32), ("frame_w", C.c_int32), ("box_top", C.c_int32),
                ("box_left", C.c_int32)]


class FcStreamDesc(C.Structure):
    _fields_ = [
        ("math", C.c_int32), ("in_dtype", C.c_int32), ("out_dtype", C.c_int32),
        ("m", C.c_int32), ("k", C.c_int32), ("ldx", C.c_int32), ("n_out", C.c_int32), ("ldo", C.c_int32),
        ("relu", C.c_int32), ("neg_slope", C.c_float),
    ]


class HeadDesc(C.Structure):
    _fields_ = [("fc", FcStreamDesc), ("hw", C.c_int32), ("pool_max", C.c_int32), ("ldp", C.c_int32)]


class AxpyDesc(C.Structure):
    _fields_ = [(f, C.c_int32) for f in ("x_dtype", "y_dtype", "out_dtype", "gate_dtype", "n", "hw", "c", "ld", "ldg",
                                         "relu")] + [("neg_slope", C.c_float), ("ax", C.c_float), ("ay", C.c_float)]


class SeGateDesc(C.Structure):
    _fields_ = [(f, C.c_int32) for f in ("dtype", "n", "hw", "c", "ld", "r", "ldg")] + [("scale", C.c_float)]


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
    "b200_conv_plan_choose": (C.c_int, [C.POINTER(ConvDesc), _i, C.POINTER(ConvPlanChoice)]),
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
    "b200_nchw_to_nhwc": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_nhwc_to_nchw": (C.c_int, [_vp, _i, _vp, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_stem_conv_out_hw": (C.c_int, [C.POINTER(StemDesc), C.POINTER(_i), C.POINTER(_i)]),
    "b200_stem_packed_weight_bytes": (_sz, [C.POINTER(StemDesc)]),
    "b200_stem_pack_weights": (C.c_int, [C.POINTER(StemDesc), _vp, _vp]),
    "b200_stem_conv_info": (C.c_int, [C.POINTER(StemDesc)] + [C.POINTER(_i)] * 5),
    "b200_stem_conv_run": (C.c_int, [C.POINTER(StemDesc), _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_stem_conv_run_image": (C.c_int, [C.POINTER(StemDesc), C.POINTER(ImageDesc), _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_image_to_nhwc": (C.c_int, [C.POINTER(ImageDesc), _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "b200_image_resize_geometry": (C.c_int, [_i, _i, _i, _i, _i] + [C.POINTER(_i)] * 4),
    "b200_image_resize_run": (C.c_int, [C.POINTER(ImageResizeDesc), _vp, _vp, _vp, _vp]),
    "b200_image_resize_geometry_ex": (C.c_int, [_i] * 6 + [C.POINTER(_i)] * 4),
    "b200_image_resize_workspace": (C.c_int, [C.POINTER(ImageResizeDesc), _i, _i, _i, _i, C.POINTER(C.c_size_t)]),
    "b200_image_resize_pil_workspace": (C.c_int, [C.POINTER(ImageResizeDesc), _i, _i, _i, C.POINTER(C.c_size_t)]),
    "b200_image_resize_pil_run": (C.c_int, [C.POINTER(ImageResizeDesc), _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "b200_image_resize_yuv_run": (C.c_int, [C.POINTER(ImageResizeDesc), _i, _vp, _vp, _vp, _vp]),
    "b200_image_resize_pil_yuv_run": (C.c_int, [C.POINTER(ImageResizeDesc), _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "b200_image_crop_resize_run": (C.c_int, [C.POINTER(ImageResizeDesc), _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp,
                                             _vp]),
    "b200_calib_stats_run": (C.c_int, [_vp, C.c_int64, _i, _i, _vp, _vp, _vp, _vp]),
    "b200_calib_kl_run": (C.c_int, [_vp, _i, _vp, _vp, _vp]),
    "b200_export_run": (C.c_int, [_vp, _i, _i, _i, _i, _i, _i, _f, _vp, _vp]),
    "b200_axpy_run": (C.c_int, [C.POINTER(AxpyDesc), _vp, _vp, _vp, _vp, _vp]),
    "b200_se_gate_workspace_bytes": (_sz, [C.POINTER(SeGateDesc)]),
    "b200_se_gate_run": (C.c_int, [C.POINTER(SeGateDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
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
    if lib.b200_abi_version() != 2:
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
