"""GPU parity for the bandwidth-bound Saber ops (pool / softmax / eltwise / activation /
scale / layout+quant transforms / depthwise conv) against the CPU oracle.
Integer results must be bit-exact; fp32 pooling / eltwise are bit-exact too (same operation
order); softmax / activation use the reference's 1e-5 default (test_saber_base.h:501)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

POOL_CASES = [
    # n, h, w, c, window, pad, stride, global
    (2, 112, 112, 64, 3, 0, 2, False),   # ResNet stem pool (ceil mode 112 -> 56)
    (1, 24, 24, 32, 2, 0, 2, False),     # VGG pool
    (3, 21, 21, 16, 3, 1, 2, False),
    (2, 13, 13, 16, 3, 1, 1, False),
    (2, 7, 7, 2048, 7, 0, 1, True),      # global average
    (1, 12, 36, 48, 3, 1, 3, False),
    (1, 17, 17, 32, 17, 0, 1, True),     # global over 289 taps: int8 leaves the SIMD kernel for the warp kernel
]


def _pool(dtype, case, ptype, x):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    lib = A.load()
    n, h, w, c, win, pad, stride, glob = case
    d = A.PoolDesc()
    d.dtype, d.type, d.n, d.h, d.w, d.c = dtype, ptype, n, h, w, c
    d.window_h = d.window_w = win
    d.pad_h = d.pad_w = pad
    d.stride_h = d.stride_w = stride
    d.global_pooling = int(glob)
    oh, ow = C.c_int32(), C.c_int32()
    A.check(lib.b200_pool_out_hw(C.byref(d), C.byref(oh), C.byref(ow)))
    xd = dev(x)
    out = torch.zeros((n, oh.value, ow.value, c), dtype=xd.dtype, device="cuda")
    A.check(lib.b200_pool_run(C.byref(d), ptr(xd), ptr(out), stream_ptr()), "pool")
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("case", POOL_CASES)
@pytest.mark.parametrize("ptype", [1, 2, 3])
def test_pool_f32(case, ptype, oracle):
    from anakin_b200 import saber_abi as A
    n, h, w, c, win, pad, stride, glob = case
    rng = np.random.default_rng(7)
    x = rng.uniform(-100, 100, (n, h, w, c)).astype(np.float32)
    want = oracle.pool_f32(x, (win, win), (pad, pad), (stride, stride), ptype, nhwc=True, global_pooling=glob)
    got = _pool(A.FLOAT, case, ptype, x)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("case", POOL_CASES)
@pytest.mark.parametrize("ptype", [1, 2, 3])
def test_pool_f16(case, ptype, oracle):
    from anakin_b200 import saber_abi as A
    n, h, w, c, win, pad, stride, glob = case
    rng = np.random.default_rng(7)
    x = rng.uniform(-100, 100, (n, h, w, c)).astype(np.float16)
    # fp32 arithmetic on the widened codes, one rounding to half at the store
    want = oracle.pool_f32(x.astype(np.float32), (win, win), (pad, pad), (stride, stride), ptype, nhwc=True,
                           global_pooling=glob).astype(np.float16)
    got = _pool(A.HALF, case, ptype, x)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("case", POOL_CASES)
@pytest.mark.parametrize("ptype", [1, 2, 3])
@pytest.mark.parametrize("unsigned", [False, True])
def test_pool_int8(case, ptype, unsigned, oracle):
    from anakin_b200 import saber_abi as A
    n, h, w, c, win, pad, stride, glob = case
    rng = np.random.default_rng(11)
    x = (rng.integers(0, 256, (n, h, w, c)).astype(np.uint8) if unsigned
         else rng.integers(-128, 128, (n, h, w, c)).astype(np.int8))
    want = oracle.pool_s8_nhwc(x, (win, win), (pad, pad), (stride, stride), ptype, global_pooling=glob)
    got = _pool(A.UINT8 if unsigned else A.INT8, case, ptype, x)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("rows,len_", [(1, 1000), (8, 1000), (32, 1000), (3, 10), (5, 4097)])
def test_softmax(rows, len_, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(3)
    x = rng.uniform(-10, 10, (rows, len_)).astype(np.float32)
    want = oracle.softmax_f32(x, rows, len_, 1)
    xd = dev(x)
    out = torch.empty_like(xd)
    A.check(A.load().b200_softmax_run(ptr(xd), ptr(out), rows, len_, 1, stream_ptr()), "softmax")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    mr, md = oracle.tensor_cmp(want, got)
    assert md < 1e-5 or mr <= 1e-5, (mr, md)
    np.testing.assert_allclose(got.sum(axis=1), 1.0, rtol=1e-5)


def test_softmax_inner(oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(4)
    x = rng.uniform(-5, 5, (3, 21, 7)).astype(np.float32)
    want = oracle.softmax_f32(x, 3, 21, 7)
    xd = dev(x)
    out = torch.empty_like(xd)
    A.check(A.load().b200_softmax_run(ptr(xd), ptr(out), 3, 21, 7, stream_ptr()))
    torch.cuda.synchronize()
    mr, md = oracle.tensor_cmp(want, out.cpu().numpy())
    assert md < 1e-5 or mr <= 1e-5


@pytest.mark.parametrize("op", [1, 2, 3])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("count", [7, 4096, 100003])
def test_eltwise_f32(op, relu, count, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(5)
    a = rng.uniform(-100, 100, count).astype(np.float32)
    b = rng.uniform(-100, 100, count).astype(np.float32)
    want = oracle.eltwise_f32(a, b, op, 0.7, -1.3, relu)
    ad, bd = dev(a), dev(b)
    out = torch.empty_like(ad)
    A.check(A.load().b200_eltwise_run(A.FLOAT, A.FLOAT, A.FLOAT, op, ptr(ad), ptr(bd), ptr(out), count,
                                      0.7, -1.3, int(relu), stream_ptr()))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), want)


@pytest.mark.parametrize("ua,ub,uo", [(False, False, False), (True, False, True), (True, True, True)])
@pytest.mark.parametrize("count", [16, 999, 65536])
def test_eltwise_int8(ua, ub, uo, count, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(6)
    mk = lambda u: (rng.integers(0, 256, count).astype(np.uint8) if u else rng.integers(-128, 128, count).astype(np.int8))
    a, b = mk(ua), mk(ub)
    dt = lambda u: A.UINT8 if u else A.INT8
    want = oracle.eltwise_sum_q8(a, b, 0.61, 0.43, dt(uo), relu=True)
    ad, bd = dev(a), dev(b)
    out = torch.zeros(count, dtype=torch.uint8 if uo else torch.int8, device="cuda")
    A.check(A.load().b200_eltwise_run(dt(ua), dt(ub), dt(uo), 2, ptr(ad), ptr(bd), ptr(out), count,
                                      0.61, 0.43, 1, stream_ptr()))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), want)


@pytest.mark.parametrize("act", [1, 2, 3, 4, 5])
def test_activation(act, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(8)
    x = rng.uniform(-6, 6, 10007).astype(np.float32)
    want = oracle.activation_f32(x, act, 0.25, 1.5)
    xd = dev(x)
    out = torch.empty_like(xd)
    A.check(A.load().b200_activation_run(A.FLOAT, act, ptr(xd), ptr(out), x.size, 0.25, 1.5, stream_ptr()))
    torch.cuda.synchronize()
    mr, md = oracle.tensor_cmp(want, out.cpu().numpy())
    assert md < 1e-5 or mr <= 1e-5, (mr, md)


def test_scale(oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(9)
    x = rng.uniform(-3, 3, (50, 24)).astype(np.float32)
    w = rng.uniform(0.5, 2, 24).astype(np.float32)
    b = rng.uniform(-1, 1, 24).astype(np.float32)
    want = oracle.scale_f32(x, 50, 24, 1, w, b)
    xd, wd, bd = dev(x), dev(w), dev(b)
    out = torch.empty_like(xd)
    A.check(A.load().b200_scale_run(A.FLOAT, ptr(xd), ptr(out), 50, 24, ptr(wd), ptr(bd), stream_ptr()))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), want)


@pytest.mark.parametrize("shape", [(2, 3, 224, 224), (1, 3, 17, 9), (2, 40, 5, 7)])
@pytest.mark.parametrize("odt", ["f32", "s8", "u8", "f16"])
def test_nchw_to_nhwc_and_back(shape, odt, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    n, c, h, w = shape
    rng = np.random.default_rng(10)
    x = rng.uniform(-1, 1, shape).astype(np.float32)
    if odt == "u8":
        x = np.abs(x)
    c_pad = (c + 15) // 16 * 16
    scale = np.float32(np.abs(x).max() / 127.0)
    xt = np.transpose(x, (0, 2, 3, 1))
    if odt == "f32":
        dtc, tdt, inv = A.FLOAT, torch.float32, 1.0
        want = xt
    elif odt == "f16":
        dtc, tdt, inv = A.HALF, torch.float16, 1.0
        want = xt.astype(np.float16)
    elif odt == "s8":
        dtc, tdt, inv = A.INT8, torch.int8, float(np.float32(1.0) / scale)
        want = oracle.quant_fp32_s8(xt, scale)
    else:
        dtc, tdt = A.UINT8, torch.uint8
        inv = float(np.float32(1.0) / (scale * np.float32(127.0 / 255.0)))
        want = oracle.quant_fp32_u8(xt, scale)
    xd = dev(x)
    out = torch.full((n, h, w, c_pad), 77, dtype=tdt, device="cuda")
    A.check(A.load().b200_nchw_to_nhwc(ptr(xd), ptr(out), dtc, n, c, h, w, c_pad, inv, 0, stream_ptr()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    np.testing.assert_array_equal(got[..., :c], want)
    assert (got[..., c:] == 0).all()
    # and back (dequantise)
    back = torch.zeros((n, c, h, w), dtype=torch.float32, device="cuda")
    A.check(A.load().b200_nhwc_to_nchw(ptr(out), dtc, ptr(back), n, c, h, w, c_pad, 1.0, stream_ptr()))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(back.cpu().numpy(), np.transpose(want.astype(np.float32), (0, 3, 1, 2)))


# (stride, filter size, dilation); 5 x 5 and dilated filters run on dwconv_vec_kernel, the 3 x 3 ones on the row kernel
DW_GEOMS = [pytest.param(1, 3, 1, id="1"), pytest.param(2, 3, 1, id="2"), pytest.param(1, 5, 1, id="5x5"),
            pytest.param(1, 3, 2, id="3x3-dil2")]


@pytest.mark.parametrize("stride,r,dil", DW_GEOMS)
def test_dwconv_f32(stride, r, dil, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(12)
    n, h, w, c = 2, 28, 28, 32
    pad = (r - 1) * dil // 2
    x = rng.uniform(-1, 1, (n, h, w, c)).astype(np.float32)
    wt = rng.uniform(-1, 1, (c, 1, r, r)).astype(np.float32)
    b = rng.uniform(-1, 1, c).astype(np.float32)
    want = oracle.conv_f32_nhwc(x, wt, b, group=c, stride=(stride, stride), dil=(dil, dil), pad=(pad, pad), relu=True)
    d = A.ConvDesc()
    d.math, d.in_dtype, d.out_dtype, d.res_dtype = A.MATH_TF32, A.FLOAT, A.FLOAT, -1
    d.n, d.h, d.w, d.c, d.k, d.ldc, d.r, d.s = n, h, w, c, c, c, r, r
    d.pad_h = d.pad_w = pad
    d.stride_h = d.stride_w = stride
    d.dil_h = d.dil_w = dil
    d.relu = 1
    wrsc = np.ascontiguousarray(np.transpose(wt[:, 0], (1, 2, 0)))
    xd, wd, bd = dev(x), dev(wrsc), dev(b)
    out = torch.zeros(want.shape, dtype=torch.float32, device="cuda")
    A.check(A.load().b200_dwconv_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), None, ptr(out), stream_ptr()))
    torch.cuda.synchronize()
    mr, md = oracle.tensor_cmp(want, out.cpu().numpy())
    assert md < 1e-3 or mr <= 1e-3


@pytest.mark.parametrize("stride,r,dil", DW_GEOMS)
def test_dwconv_f16(stride, r, dil, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(13)
    n, h, w, c = 2, 30, 26, 48
    pad = (r - 1) * dil // 2
    x = rng.uniform(-1, 1, (n, h, w, c)).astype(np.float16)
    wt = rng.uniform(-1, 1, (c, 1, r, r)).astype(np.float16)
    b = rng.uniform(-1, 1, c).astype(np.float32)
    want = oracle.conv_f32_nhwc(x.astype(np.float32), wt.astype(np.float32), b, group=c, stride=(stride, stride), dil=(dil, dil), pad=(pad, pad),
                                relu=True)
    d = A.ConvDesc()
    d.math, d.in_dtype, d.out_dtype, d.res_dtype = A.MATH_F16, A.HALF, A.HALF, -1
    d.n, d.h, d.w, d.c, d.k, d.ldc, d.r, d.s = n, h, w, c, c, c, r, r
    d.pad_h = d.pad_w = pad
    d.stride_h = d.stride_w = stride
    d.dil_h = d.dil_w = dil
    d.relu = 1
    wrsc = np.ascontiguousarray(np.transpose(wt[:, 0], (1, 2, 0)))
    xd, wd, bd = dev(x), dev(wrsc), dev(b)
    out = torch.zeros(want.shape, dtype=torch.float16, device="cuda")
    A.check(A.load().b200_dwconv_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), None, ptr(out), stream_ptr()))
    torch.cuda.synchronize()
    # fp32 accumulation of exact products, one rounding to half at the store
    np.testing.assert_array_equal(out.cpu().numpy(), want.astype(np.float16))


@pytest.mark.parametrize("stride,r,dil", DW_GEOMS)
@pytest.mark.parametrize("variant", ["u8_relu_u8", "s8_s8", "u8_s8"])
def test_dwconv_int8_bit_exact(stride, r, dil, variant, oracle):
    """INT8 depthwise (SaberDepthWiseConv's int8 arm, saber_depthwiseconv_act.cu:84-295): exact s32 sums, then the x86
    Saber epilogue -- bit-identical to the grouped x86 oracle (pinned to conv_basic_check_int8 with group = c)."""
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(abs(hash((stride, variant))) % (2 ** 31))
    n, h, w, c = 2, 29, 31, 96
    pad = (r - 1) * dil // 2
    in_u = variant.startswith("u8")
    x = rng.integers(0, 256, (n, h, w, c)).astype(np.uint8) if in_u else rng.integers(-128, 128, (n, h, w, c)).astype(np.int8)
    wq = rng.integers(-127, 128, (c, 1, r, r)).astype(np.int8)
    bias = rng.uniform(-3000, 3000, c).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, c).astype(np.float32) * np.float32(1.0 / 900.0)
    out_dtype = A.UINT8 if variant.endswith("relu_u8") else A.INT8
    relu = variant.endswith("relu_u8")
    want = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, out_dtype=out_dtype, stride=(stride, stride), dil=(dil, dil), pad=(pad, pad), relu=relu,
                                   group=c)
    d = A.ConvDesc()
    d.math, d.in_dtype, d.out_dtype, d.res_dtype = A.MATH_I8, (A.UINT8 if in_u else A.INT8), out_dtype, -1
    d.n, d.h, d.w, d.c, d.k, d.ldc, d.r, d.s = n, h, w, c, c, c, r, r
    d.pad_h = d.pad_w = pad
    d.stride_h = d.stride_w = stride
    d.dil_h = d.dil_w = dil
    d.relu = int(relu)
    wrsc = np.ascontiguousarray(np.transpose(wq[:, 0], (1, 2, 0)))
    xd, wd, bd, sd = dev(x), dev(wrsc), dev(bias), dev(scale)
    out = torch.zeros(want.shape, dtype=(torch.uint8 if out_dtype == A.UINT8 else torch.int8), device="cuda")
    A.check(A.load().b200_dwconv_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), ptr(sd), ptr(out), stream_ptr()))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), want)


# shapes that take the shared-memory tiled kernel (3x3 / stride 1, >= 28 x 28 outputs for the float kinds): 8, 4 and 2 channel vectors per
# block, several channel blocks, ragged tiles in both directions, with and without padding
DW_TILE_CASES = [  # (n, h, w, vectors of 16 B per pixel, pad)
    (2, 30, 37, 8, 1), (1, 29, 70, 4, 1), (1, 40, 120, 2, 1), (1, 56, 56, 16, 1), (2, 34, 45, 8, 0), (1, 31, 66, 4, 0),
    # more tiles than co-resident blocks (3 x 148): several waves of blocks
    (112, 28, 28, 8, 1), (112, 28, 60, 4, 1),
]


@pytest.mark.parametrize("case", DW_TILE_CASES)
@pytest.mark.parametrize("kind", ["f32", "f16", "u8_relu_u8", "s8_s8"])
def test_dwconv_tiled(case, kind, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    n, h, w, cv, pad = case
    rng = np.random.default_rng(abs(hash((case, kind))) % (2 ** 31))
    d = A.ConvDesc()
    d.res_dtype = -1
    d.r = d.s = 3
    d.pad_h = d.pad_w = pad
    d.stride_h = d.stride_w = d.dil_h = d.dil_w = 1
    sd = None
    if kind in ("f32", "f16"):
        np_t, es = (np.float32, 4) if kind == "f32" else (np.float16, 2)
        c = cv * 16 // es
        x = rng.uniform(-1, 1, (n, h, w, c)).astype(np_t)
        wt = rng.uniform(-1, 1, (c, 1, 3, 3)).astype(np_t)
        b = rng.uniform(-1, 1, c).astype(np.float32)
        want = oracle.conv_f32_nhwc(x.astype(np.float32), wt.astype(np.float32), b, group=c, pad=(pad, pad), relu=True, neg_slope=0.1)
        d.math, d.in_dtype, d.out_dtype = (A.MATH_TF32, A.FLOAT, A.FLOAT) if kind == "f32" else (A.MATH_F16, A.HALF, A.HALF)
        d.relu, d.neg_slope = 1, 0.1
        tdt = torch.float32 if kind == "f32" else torch.float16
    else:
        c = cv * 16
        in_u = kind.startswith("u8")
        x = rng.integers(0, 256, (n, h, w, c)).astype(np.uint8) if in_u else rng.integers(-128, 128, (n, h, w, c)).astype(np.int8)
        wt = rng.integers(-127, 128, (c, 1, 3, 3)).astype(np.int8)
        b = rng.uniform(-3000, 3000, c).astype(np.float32)
        scale = rng.uniform(0.5, 1.5, c).astype(np.float32) * np.float32(1.0 / 900.0)
        relu = kind.endswith("relu_u8")
        out_dtype = A.UINT8 if relu else A.INT8
        want = oracle.conv_s8_nhwc_x86(x, wt, b, scale, out_dtype=out_dtype, pad=(pad, pad), relu=relu, group=c)
        d.math, d.in_dtype, d.out_dtype = A.MATH_I8, (A.UINT8 if in_u else A.INT8), out_dtype
        d.relu = int(relu)
        sd = dev(scale)
        tdt = torch.uint8 if relu else torch.int8
    d.n, d.h, d.w, d.c, d.k, d.ldc = n, h, w, c, c, c
    wrsc = np.ascontiguousarray(np.transpose(wt[:, 0], (1, 2, 0)))
    xd, wd, bd = dev(x), dev(wrsc), dev(b)
    out = torch.zeros(want.shape, dtype=tdt, device="cuda")
    A.check(A.load().b200_dwconv_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), ptr(sd), ptr(out), stream_ptr()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    if kind == "f32":
        mr, md = oracle.tensor_cmp(want, got)
        assert md < 1e-3 or mr <= 1e-3
        assert np.abs(got - want).max() <= 1e-5        # 9 fp32 FMAs against the oracle's fp32 sum
    elif kind == "f16":
        np.testing.assert_array_equal(got, want.astype(np.float16))   # fp32 accumulation, one rounding at the store
    else:
        np.testing.assert_array_equal(got, want)


# ---------------------------------------------------------------------------------------------------------------
# Weight-streaming inner product (fc_stream.cu) and the fused classifier head (pool + fc + softmax, one launch)
FC_CASES = [(8, 2048, 1000), (4, 25088, 512), (1, 512, 10), (13, 4096, 200), (16, 1024, 64)]   # (m, k, n)


@pytest.mark.parametrize("m,k,n", FC_CASES)
@pytest.mark.parametrize("variant", ["u8_f32", "s8_relu_u8", "u8_s8"])
def test_fc_stream_int8_bit_exact(m, k, n, variant, oracle):
    """int8 inner product: exact dp4a sums + the x86 Saber epilogue, bit-identical to the 1x1-conv oracle."""
    import ctypes as C
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(hash((m, k, n, variant)) % (2 ** 31))
    unsigned = variant.startswith("u8")
    x = (rng.integers(0, 256, (m, 1, 1, k)).astype(np.uint8) if unsigned else rng.integers(-128, 128, (m, 1, 1, k)).astype(np.int8))
    w = rng.integers(-127, 128, (n, k, 1, 1)).astype(np.int8)
    bias = rng.uniform(-2000, 2000, n).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, n).astype(np.float32) * np.float32(1.0 / (40.0 * np.sqrt(k) * 8))
    out_dtype = {"u8_f32": A.FLOAT, "s8_relu_u8": A.UINT8, "u8_s8": A.INT8}[variant]
    relu = variant == "s8_relu_u8"
    want = oracle.conv_s8_nhwc_x86(x, w, bias, scale, out_dtype=out_dtype, relu=relu).reshape(m, n)
    lib = A.load()
    d = A.FcStreamDesc()
    d.math, d.in_dtype, d.out_dtype = A.MATH_I8, (A.UINT8 if unsigned else A.INT8), out_dtype
    d.m, d.k, d.ldx, d.n_out = m, k, k, n
    d.ldo = (n + 15) // 16 * 16
    d.relu = int(relu)
    out = torch.zeros((m, d.ldo), dtype={A.FLOAT: torch.float32, A.UINT8: torch.uint8, A.INT8: torch.int8}[out_dtype], device="cuda")
    xd, wd, bd, sd = dev(x.reshape(m, k)), dev(w.reshape(n, k)), dev(bias), dev(scale)
    assert m <= lib.b200_fc_stream_max_rows()
    A.check(lib.b200_fc_stream_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), ptr(sd), ptr(out), stream_ptr()), "fc_stream")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert (got[:, n:] == 0).all()
    np.testing.assert_array_equal(got[:, :n], want)


@pytest.mark.parametrize("m,k,n", [(4, 25088, 256), (8, 1024, 1000), (3, 4096, 100)])
@pytest.mark.parametrize("math", ["f32", "f16"])
def test_fc_stream_float(m, k, n, math, oracle):
    import ctypes as C
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(hash((m, k, n, math)) % (2 ** 31))
    x = rng.uniform(-1, 1, (m, k)).astype(np.float32)
    w = (rng.standard_normal((n, k)) * np.sqrt(2.0 / k)).astype(np.float32)
    bias = rng.uniform(-0.5, 0.5, n).astype(np.float32)
    if math == "f16":
        xs, ws = x.astype(np.float16), w.astype(np.float16)
        x_seen, w_seen = xs.astype(np.float32), ws.astype(np.float32)
        mk, dt = A.MATH_F16, A.HALF
    else:
        xs, ws, x_seen, w_seen = x, w, x, w
        mk, dt = A.MATH_TF32X3, A.FLOAT
    want = np.maximum(x_seen.astype(np.float64) @ w_seen.astype(np.float64).T + bias, 0).astype(np.float32)
    lib = A.load()
    d = A.FcStreamDesc()
    d.math, d.in_dtype, d.out_dtype = mk, dt, A.FLOAT
    d.m, d.k, d.ldx, d.n_out, d.ldo, d.relu = m, k, k, n, n, 1
    out = torch.zeros((m, n), dtype=torch.float32, device="cuda")
    xd, wd, bd = dev(xs), dev(ws), dev(bias)
    A.check(lib.b200_fc_stream_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), None, ptr(out), stream_ptr()), "fc_stream")
    torch.cuda.synchronize()
    mr, md = oracle.tensor_cmp(want, out.cpu().numpy())
    assert md < 1e-3 or mr <= 1e-3, (mr, md)
    assert md <= 2e-5 * max(1.0, float(np.abs(want).max())) * max(1.0, k / 4096), md


@pytest.mark.parametrize("m,hw,c,n", [(8, 49, 2048, 1000), (2, 49, 512, 10), (5, 16, 1024, 257), (1, 49, 2048, 1000),
                                      (8, 4, 64, 33)])
@pytest.mark.parametrize("dtype", ["u8", "s8"])
@pytest.mark.parametrize("pool", ["avg", "max"])
def test_fused_head_matches_the_three_separate_ops(m, hw, c, n, dtype, pool, oracle):
    """b200_head_run == b200_pool_run -> b200_fc_stream_run -> b200_softmax_rows on every tensor it writes, bit for
    bit, over repeated launches on the same (self-cleaning) workspace; the pooled codes are the oracle's."""
    import ctypes as C
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(hash((m, hw, c, n, dtype, pool)) % (2 ** 31))
    lib = A.load()
    side = int(round(hw ** 0.5))
    assert side * side == hw
    if dtype == "u8":
        x = rng.integers(0, 256, (m, side, side, c)).astype(np.uint8)
        dt, tdt = A.UINT8, torch.uint8
    else:
        x = rng.integers(-128, 128, (m, side, side, c)).astype(np.int8)
        dt, tdt = A.INT8, torch.int8
    w = rng.integers(-127, 128, (n, c)).astype(np.int8)
    scale = rng.uniform(0.5, 1.5, n).astype(np.float32) * np.float32(1.0 / (40.0 * np.sqrt(c) * 8))
    bias = rng.uniform(-2000, 2000, n).astype(np.float32)
    xd, wd, bd, sd = dev(x), dev(w), dev(bias), dev(scale)
    ldo = (n + 3) // 4 * 4
    # --- the three separate ops
    pd = A.PoolDesc()
    pd.dtype, pd.type, pd.n, pd.h, pd.w, pd.c = dt, (A.POOL_MAX if pool == "max" else A.POOL_AVG_INC), m, side, side, c
    pd.window_h = pd.window_w = side
    pd.stride_h = pd.stride_w = 1
    pd.global_pooling = 1
    pooled_ref = torch.zeros((m, c), dtype=tdt, device="cuda")
    A.check(lib.b200_pool_run(C.byref(pd), ptr(xd), ptr(pooled_ref), stream_ptr()), "pool")
    fd = A.FcStreamDesc()
    fd.math, fd.in_dtype, fd.out_dtype = A.MATH_I8, dt, A.FLOAT
    fd.m, fd.k, fd.ldx, fd.n_out, fd.ldo = m, c, c, n, ldo
    logits_ref = torch.zeros((m, ldo), dtype=torch.float32, device="cuda")
    A.check(lib.b200_fc_stream_run(C.byref(fd), ptr(pooled_ref), ptr(wd), ptr(bd), ptr(sd), ptr(logits_ref), stream_ptr()), "fc")
    prob_ref = torch.zeros((m, ldo), dtype=torch.float32, device="cuda")
    A.check(lib.b200_softmax_rows(ptr(logits_ref), ptr(prob_ref), m, n, ldo, ldo, stream_ptr()), "softmax")
    # --- one launch
    hd = A.HeadDesc()
    hd.fc, hd.hw, hd.pool_max, hd.ldp = fd, hw, int(pool == "max"), ldo
    pooled = torch.zeros((m, c), dtype=tdt, device="cuda")
    logits = torch.zeros((m, ldo), dtype=torch.float32, device="cuda")
    prob = torch.zeros((m, ldo), dtype=torch.float32, device="cuda")
    ws = torch.zeros(lib.b200_head_workspace_bytes(C.byref(hd)), dtype=torch.uint8, device="cuda")
    for rep in range(3):
        A.check(lib.b200_head_run(C.byref(hd), ptr(xd), ptr(pooled), ptr(wd), ptr(bd), ptr(sd), ptr(logits), ptr(prob),
                                  ptr(ws), stream_ptr()), "head")
        torch.cuda.synchronize()
        assert torch.equal(pooled, pooled_ref), rep
        assert torch.equal(logits, logits_ref), rep
        assert torch.equal(prob, prob_ref), rep
        assert int(ws.count_nonzero()) == 0, "the workspace must be left zeroed"
    want_pool = oracle.pool_s8_nhwc(x, (side, side), (0, 0), (side, side), 1 if pool == "max" else 2, global_pooling=True)
    np.testing.assert_array_equal(pooled.cpu().numpy(), want_pool.reshape(m, c))
    np.testing.assert_allclose(prob.cpu().numpy()[:, :n].sum(1), 1.0, rtol=1e-5)
    # float heads are not fused: the entry point says so and the Net keeps the three ops
    fd.math, fd.in_dtype = A.MATH_F16, A.HALF
    hd.fc = fd
    assert lib.b200_head_run(C.byref(hd), ptr(xd), ptr(pooled), ptr(wd), ptr(bd), ptr(sd), ptr(logits), ptr(prob), ptr(ws),
                             stream_ptr()) == A.UNIMPL_ERROR
