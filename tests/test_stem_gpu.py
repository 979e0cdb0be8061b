"""GPU parity: the stem kernel (conv_stem.cu: graph-input conv + relu [+ max pool] in one launch, C ABI
b200_stem_conv_*) vs the CPU oracle.

INT8: fp32 NCHW input quantised with the x86 rule (oracle.quant_fp32_s8), conv_s8_nhwc_x86, then -- fused --
pool_s8_nhwc: bit-exact, as saber_conv_pooling.cpp's conv -> pool is (max commutes with the requantisation).
Float kinds: the reference criterion of test_saber_base.h:470 (tensor_cmp_host), against conv_f32_nhwc o pool_f32 on
the operand values the tensor core sees. Shapes: the ResNet-50 / MobileNet / VGG16 stems, ragged tiles, padded and
ceil-mode pooling windows, stride 1 and 2, 1..4 input channels, output channel counts below / above one tile.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (n, c, h, w, k, r, s, stride, pad, pool) ; pool = None | (window, stride, pad)
STEM_CASES = [
    (2, 3, 224, 224, 64, 7, 7, 2, 3, (3, 2, 0)),     # ResNet-50 conv1 + pool1 (ceil mode 112 -> 56)
    (1, 3, 224, 224, 64, 7, 7, 2, 3, None),          # the conv alone
    (2, 3, 64, 64, 32, 3, 3, 2, 1, None),            # MobileNet conv1 shape, k = 32
    (1, 3, 48, 40, 64, 3, 3, 1, 1, (2, 2, 0)),       # VGG-like 3x3/s1 + 2x2/s2
    (3, 3, 37, 45, 64, 7, 7, 2, 3, (3, 2, 0)),       # ragged everything
    (1, 3, 33, 33, 16, 5, 5, 2, 2, (3, 2, 1)),       # padded pooling window, k = 16
    (2, 1, 30, 30, 48, 3, 3, 1, 0, (2, 2, 0)),       # one input channel, k = 48 (padded to 64 in the tile)
    (1, 4, 20, 28, 128, 3, 3, 1, 1, None),           # four channels, two n-tiles
    (1, 3, 56, 56, 80, 7, 7, 2, 3, (3, 2, 0)),       # two n-tiles, the second ragged
]


def _stem_desc(A, math, out_dtype, case, ldc, relu, inv_scale, neg_slope=0.0, monotone=0):
    n, c, h, w, k, r, s, stride, pad, pool = case
    d = A.StemDesc()
    d.math, d.out_dtype = math, out_dtype
    d.n, d.c, d.h, d.w, d.k, d.ldc = n, c, h, w, k, ldc
    d.r, d.s, d.stride_h, d.stride_w, d.pad_h, d.pad_w = r, s, stride, stride, pad, pad
    d.relu, d.neg_slope, d.in_inv_scale = int(relu), neg_slope, inv_scale
    d.monotone_epilogue = monotone
    if pool is not None:
        d.fuse_pool, d.pool_type = 1, A.POOL_MAX
        d.pool_window_h = d.pool_window_w = pool[0]
        d.pool_stride_h = d.pool_stride_w = pool[1]
        d.pool_pad_h = d.pool_pad_w = pool[2]
    return d


def _run_stem(A, d, x_nchw, w_operand, bias, scale, np_out, fill=0):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    lib = A.load()
    oh, ow = C.c_int32(), C.c_int32()
    A.check(lib.b200_stem_conv_out_hw(C.byref(d), C.byref(oh), C.byref(ow)), "stem_out_hw")
    packed = np.zeros(lib.b200_stem_packed_weight_bytes(C.byref(d)), np.uint8)
    wsrc = np.ascontiguousarray(w_operand)
    A.check(lib.b200_stem_pack_weights(C.byref(d), wsrc.ctypes.data_as(C.c_void_p), packed.ctypes.data_as(C.c_void_p)), "stem_pack")
    xd, wd = dev(x_nchw), dev(packed)
    bd = dev(bias) if bias is not None else None
    sd = dev(scale) if scale is not None else None
    out = torch.full((d.n, oh.value, ow.value, d.ldc), fill, dtype=np_out, device="cuda")
    A.check(lib.b200_stem_conv_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), ptr(sd), ptr(out), stream_ptr()), "stem_run")
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("case", STEM_CASES)
@pytest.mark.parametrize("variant", ["relu_u8", "s8", "f32"])
@pytest.mark.parametrize("monotone", [0, 1])     # 1: the fused pooling runs on the raw accumulators (positive scales)
def test_stem_int8_bit_exact(case, variant, monotone, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    rng = np.random.default_rng(abs(hash((case, variant))) % (2 ** 31))
    n, c, h, w, k, r, s, stride, pad, pool = case
    x = rng.uniform(-2.6, 2.6, (n, c, h, w)).astype(np.float32)
    in_scale = np.float32(2.64 / 127.0)
    wq = rng.integers(-127, 128, (k, c, r, s)).astype(np.int8)
    bias = rng.uniform(-2000, 2000, k).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, k).astype(np.float32) * np.float32(1.0 / (40.0 * np.sqrt(c * r * s) * 8))
    out_dtype = {"relu_u8": A.UINT8, "s8": A.INT8, "f32": A.FLOAT}[variant]
    relu = variant == "relu_u8"
    xq = oracle.quant_fp32_s8(np.ascontiguousarray(x.transpose(0, 2, 3, 1)), in_scale)
    want = oracle.conv_s8_nhwc_x86(xq, wq, bias, scale, out_dtype=out_dtype, stride=(stride, stride), pad=(pad, pad), relu=relu)
    if pool is not None:
        if out_dtype == A.FLOAT:
            want = oracle.pool_f32(want, (pool[0],) * 2, (pool[2],) * 2, (pool[1],) * 2, A.POOL_MAX, nhwc=True)
        else:
            want = oracle.pool_s8_nhwc(want, (pool[0],) * 2, (pool[2],) * 2, (pool[1],) * 2, A.POOL_MAX)
    ldc = (k + 15) // 16 * 16 + (16 if variant == "s8" else 0)     # one case family with a row pitch above k
    if out_dtype == A.FLOAT:
        ldc = (k + 3) // 4 * 4
    if monotone and pool is None:
        pytest.skip("the flag only matters with a fused pooling")
    d = _stem_desc(A, A.MATH_I8, out_dtype, case, ldc, relu, float(np.float32(1.0) / in_scale), monotone=monotone)
    tdt = {A.UINT8: torch.uint8, A.INT8: torch.int8, A.FLOAT: torch.float32}[out_dtype]
    got = _run_stem(A, d, x, wq, bias, scale, tdt)
    assert (got[..., k:] == 0).all(), "padding channels must stay untouched"
    got = got[..., :k]
    assert got.shape == want.shape, (got.shape, want.shape)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("case", [STEM_CASES[0], STEM_CASES[2], STEM_CASES[3], STEM_CASES[4], STEM_CASES[7]])
@pytest.mark.parametrize("math", ["f16", "tf32x3"])
@pytest.mark.parametrize("monotone", [0, 1])
def test_stem_float(case, math, monotone, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    rng = np.random.default_rng(abs(hash((case, math))) % (2 ** 31))
    n, c, h, w, k, r, s, stride, pad, pool = case
    x = rng.uniform(-1, 1, (n, c, h, w)).astype(np.float32)
    wt = (rng.standard_normal((k, c, r, s)) * np.sqrt(2.0 / (c * r * s))).astype(np.float32)
    bias = rng.uniform(-0.5, 0.5, k).astype(np.float32)
    if math == "f16":
        w_op = wt.astype(np.float16)
        x_seen, w_seen = x.astype(np.float16).astype(np.float32), w_op.astype(np.float32)
        mk, out_dtype, tdt = A.MATH_F16, A.HALF, torch.float16
    else:
        w_op, x_seen, w_seen = wt, x, wt
        mk, out_dtype, tdt = A.MATH_TF32X3, A.FLOAT, torch.float32
    want = oracle.conv_f32_nhwc(np.ascontiguousarray(x_seen.transpose(0, 2, 3, 1)), w_seen, bias, stride=(stride, stride),
                                pad=(pad, pad), relu=True, neg_slope=0.1)
    if out_dtype == A.HALF:
        want = want.astype(np.float16).astype(np.float32)     # the conv output edge is stored in half
    if pool is not None:
        want = oracle.pool_f32(want, (pool[0],) * 2, (pool[2],) * 2, (pool[1],) * 2, A.POOL_MAX, nhwc=True)
    if monotone and pool is None:
        pytest.skip("the flag only matters with a fused pooling")
    d = _stem_desc(A, mk, out_dtype, case, k, True, 1.0, neg_slope=0.1, monotone=monotone)
    got = _run_stem(A, d, x, w_op, bias, None, tdt).astype(np.float32)
    assert got.shape == want.shape, (got.shape, want.shape)
    max_ratio, max_diff = oracle.tensor_cmp(want, got)
    tol = 2e-3 if math == "f16" else 1e-3      # f16: one half ulp of the stored edge on top of the criterion
    assert max_diff < tol or max_ratio <= tol, (max_ratio, max_diff)
    if math == "tf32x3":
        assert max_diff <= 2e-5 * max(1.0, float(np.abs(want).max())), max_diff


def test_stem_rejects_what_it_cannot_fuse():
    from anakin_b200 import saber_abi as A
    lib = A.load()
    case = (1, 3, 32, 32, 64, 3, 3, 1, 1, (2, 2, 0))
    d = _stem_desc(A, A.MATH_I8, A.UINT8, case, 64, True, 1.0)
    d.pool_type = A.POOL_AVG_EXC
    oh, ow = C.c_int32(), C.c_int32()
    assert lib.b200_stem_conv_out_hw(C.byref(d), C.byref(oh), C.byref(ow)) == A.UNIMPL_ERROR
    d = _stem_desc(A, A.MATH_I8, A.UINT8, (1, 8, 32, 32, 64, 3, 3, 1, 1, None), 64, True, 1.0)
    assert lib.b200_stem_conv_out_hw(C.byref(d), C.byref(oh), C.byref(ow)) == A.INVALID_VALUE
