"""GPU parity: wgmma implicit-GEMM conv (C ABI) vs the CPU oracle.

INT8 must be bit-exact against oracle_conv_s8_nhwc_x86 (x86 Saber semantics). Float
kinds are checked with the reference's own criterion (test_saber_base.h:470 with
tensor_cmp_host: max_diff < 1e-3 or max_ratio <= 1e-3) against conv_basic_check semantics
evaluated on the operand values the tensor core sees (f16-rounded inputs; 3xTF32 on the fp32 inputs themselves).
Shape sweep follows test/saber/test_saber_conv.cpp:868-901,1000-1015 plus the ResNet-50
layer shapes of SURVEY.md section 8d.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (n, h, w, c, k, r, stride, pad, dil)
I8_CASES = [
    (2, 12, 12, 64, 64, 1, 1, 0, 1),
    (1, 21, 21, 128, 32, 1, 1, 0, 1),
    (3, 12, 12, 64, 64, 3, 1, 1, 1),
    (1, 24, 24, 32, 40, 3, 2, 1, 1),
    (2, 14, 14, 256, 256, 3, 1, 1, 1),
    (1, 36, 36, 16, 64, 3, 1, 1, 2),
    (2, 56, 56, 64, 256, 1, 1, 0, 1),
    (2, 56, 56, 256, 128, 1, 2, 0, 1),
    (1, 7, 7, 512, 2048, 1, 1, 0, 1),
    (8, 7, 7, 512, 512, 3, 1, 1, 1),
    (1, 64, 64, 16, 64, 7, 2, 3, 1),   # stem-like, 3 real channels padded to 16
    (8, 1, 1, 2048, 1000, 1, 1, 0, 1),  # fc as 1x1 conv, ragged N
]


def _mk_i8(rng, case, in_unsigned):
    n, h, w, c, k, r, stride, pad, dil = case
    c_real = 3 if (r == 7) else c
    if in_unsigned:
        x = rng.integers(0, 256, (n, h, w, c_real)).astype(np.uint8)
    else:
        x = rng.integers(-128, 128, (n, h, w, c_real)).astype(np.int8)
    wq = rng.integers(-127, 128, (k, c_real, r, r)).astype(np.int8)
    bias = rng.uniform(-2000, 2000, k).astype(np.float32)
    kk = c_real * r * r
    scale = rng.uniform(0.5, 1.5, k).astype(np.float32) * np.float32(1.0 / (40.0 * np.sqrt(kk) * 8))
    return x, wq, bias, scale


@pytest.mark.parametrize("case", I8_CASES)
@pytest.mark.parametrize("variant", ["s8_relu_u8", "u8_res_s8", "s8_f32"])
def test_conv_int8_bit_exact(case, variant, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev, pad_channels
    rng = np.random.default_rng(hash((case, variant)) % (2 ** 31))
    n, h, w, c, k, r, stride, pad, dil = case
    in_unsigned = variant == "u8_res_s8"
    x, wq, bias, scale = _mk_i8(rng, case, in_unsigned)
    out_dtype = {"s8_relu_u8": A.UINT8, "u8_res_s8": A.INT8, "s8_f32": A.FLOAT}[variant]
    relu = variant != "s8_f32"
    kw = dict(stride=(stride, stride), pad=(pad, pad), dil=(dil, dil), relu=relu)
    res = None
    sum_scale = 1.0
    oh = oracle.conv_out_size(h, pad, dil, r, stride)
    if variant == "u8_res_s8":
        res = rng.integers(0, 256, (n, oh, oh, k)).astype(np.uint8)
        sum_scale = 0.37
    want = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, residual=res, sum_scale=sum_scale,
                                   out_dtype=out_dtype, **kw)
    xin = pad_channels(x, c)
    # output / residual rows are padded to a 16-byte multiple, as the framework's NHWC tensors are
    ldc = (k + 15) // 16 * 16 if out_dtype != A.FLOAT else (k + 3) // 4 * 4
    run = ConvRunner(A.MATH_I8, xin.shape, A.UINT8 if in_unsigned else A.INT8, wq, bias, scale,
                     out_dtype, res_dtype=(A.UINT8 if res is not None else -1), sum_scale=sum_scale, ldc=ldc, **kw)
    got = run.run(dev(xin), dev(pad_channels(res, ldc)) if res is not None else None)
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    assert (got[..., k:] == 0).all(), "padding channels must stay untouched"
    got = got[..., :k]
    assert got.shape == want.shape
    if out_dtype == A.FLOAT:
        np.testing.assert_array_equal(got, want)
    else:
        bad = np.argwhere(got != want)
        assert bad.shape[0] == 0, "first mismatches %s (info %s)" % (bad[:5], run.info())


# split-K (cluster of `split` CTAs along the k loop, reduce-scatter of the partial sums through distributed
# shared memory) under forced tile widths: every slice / ragged-channel combination must stay bit-exact.
SPLIT_CASES = [
    # (case, BN, split)
    ((2, 7, 7, 512, 512, 3, 1, 1, 1), 32, 2),
    ((2, 7, 7, 512, 512, 3, 1, 1, 1), 64, 4),
    ((2, 7, 7, 512, 512, 3, 1, 1, 1), 128, 8),
    ((1, 14, 14, 256, 200, 3, 1, 1, 1), 128, 4),   # second n tile: slices with 32, 32, 8 and 0 real channels
    ((1, 14, 14, 256, 200, 3, 1, 1, 1), 64, 2),
    ((3, 7, 7, 2048, 72, 1, 1, 0, 1), 128, 8),     # 16-channel slices, most of them empty
    ((1, 9, 9, 1024, 1000, 1, 1, 0, 1), 128, 2),
]


@pytest.mark.parametrize("case,bn,split", SPLIT_CASES)
@pytest.mark.parametrize("variant", ["s8_relu_u8", "u8_res_s8", "s8_f32"])
def test_conv_int8_split_k_bit_exact(case, bn, split, variant, oracle, monkeypatch):
    monkeypatch.setenv("B200_SABER_FORCE_BN", str(bn))
    monkeypatch.setenv("B200_SABER_FORCE_SPLIT", str(split))
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev, pad_channels
    rng = np.random.default_rng(hash((case, bn, split, variant)) % (2 ** 31))
    n, h, w, c, k, r, stride, pad, dil = case
    in_unsigned = variant == "u8_res_s8"
    x, wq, bias, scale = _mk_i8(rng, case, in_unsigned)
    out_dtype = {"s8_relu_u8": A.UINT8, "u8_res_s8": A.INT8, "s8_f32": A.FLOAT}[variant]
    kw = dict(stride=(stride, stride), pad=(pad, pad), dil=(dil, dil), relu=variant != "s8_f32")
    res, sum_scale = None, 1.0
    oh = oracle.conv_out_size(h, pad, dil, r, stride)
    if variant == "u8_res_s8":
        res = rng.integers(0, 256, (n, oh, oh, k)).astype(np.uint8)
        sum_scale = 0.37
    want = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, residual=res, sum_scale=sum_scale, out_dtype=out_dtype, **kw)
    ldc = (k + 15) // 16 * 16 if out_dtype != A.FLOAT else (k + 3) // 4 * 4
    run = ConvRunner(A.MATH_I8, x.shape, A.UINT8 if in_unsigned else A.INT8, wq, bias, scale,
                     out_dtype, res_dtype=(A.UINT8 if res is not None else -1), sum_scale=sum_scale, ldc=ldc, **kw)
    info = run.info()
    if out_dtype == A.FLOAT and bn > 128:
        pytest.skip("4-byte outputs cap the tile at 128 channels")
    assert info["block_n"] == bn and info["split"] == split, info
    got = run.run(dev(x), dev(pad_channels(res, ldc)) if res is not None else None)
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    assert (got[..., k:] == 0).all(), "padding channels must stay untouched"
    np.testing.assert_array_equal(got[..., :k], want)


F_CASES = [
    (1, 12, 12, 16, 32, 3, 1, 1, 1),
    (3, 21, 21, 8, 8, 3, 2, 1, 1),
    (2, 24, 24, 64, 64, 1, 1, 0, 1),
    (1, 36, 36, 32, 48, 3, 1, 2, 2),
    (2, 28, 28, 128, 128, 3, 1, 1, 1),
    (1, 56, 56, 64, 64, 1, 2, 0, 1),
    (1, 40, 40, 4, 64, 7, 2, 3, 1),   # stem-like (3 real channels)
]


@pytest.mark.parametrize("math", ["f16", "tf32x3"])
@pytest.mark.parametrize("bn,split", [(32, 2), (64, 4), (128, 4)])
def test_conv_float_split_k(math, bn, split, oracle, monkeypatch):
    """float kinds through the split-K cluster path (fp32 partial sums, fixed summation order)."""
    monkeypatch.setenv("B200_SABER_FORCE_BN", str(bn))
    monkeypatch.setenv("B200_SABER_FORCE_SPLIT", str(split))
    test_conv_float((2, 14, 14, 128, 200, 3, 1, 1, 1), math, True, oracle, expect=(bn, split))


@pytest.mark.parametrize("case", F_CASES)
@pytest.mark.parametrize("math", ["f16", "tf32x3"])
@pytest.mark.parametrize("with_res", [False, True])
def test_conv_float(case, math, with_res, oracle, expect=None):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev, pad_channels
    rng = np.random.default_rng(hash((case, math, with_res)) % (2 ** 31))
    n, h, w, c, k, r, stride, pad, dil = case
    if math == "f16" and c % 8:
        c = 8
    c_real = 3 if r == 7 else c
    x = rng.uniform(-1, 1, (n, h, w, c_real)).astype(np.float32)
    wt = (rng.standard_normal((k, c_real, r, r)) * np.sqrt(2.0 / (c_real * r * r))).astype(np.float32)
    bias = rng.uniform(-0.5, 0.5, k).astype(np.float32)
    kw = dict(stride=(stride, stride), pad=(pad, pad), dil=(dil, dil), relu=True, neg_slope=0.1)
    oh = oracle.conv_out_size(h, pad, dil, r, stride)
    res = rng.uniform(-1, 1, (n, oh, oh, k)).astype(np.float32) if with_res else None
    if math == "f16":
        xs, ws = x.astype(np.float16), wt.astype(np.float16)
        x_seen, w_seen = xs.astype(np.float32), ws.astype(np.float32)
        mk, dt = A.MATH_F16, A.HALF
        res_in = res.astype(np.float16) if with_res else None
        res_seen = res_in.astype(np.float32) if with_res else None
    else:
        # error-compensated split: compare against the exact-fp32 operands, fp32-grade tolerance
        xs, ws = x, wt
        x_seen, w_seen = x, wt
        mk, dt = A.MATH_TF32X3, A.FLOAT
        res_in = res
        res_seen = res
    want = oracle.conv_f32_nhwc(x_seen, w_seen, bias, residual=res_seen, beta=1.0, **kw)
    xin = pad_channels(xs, c)
    run = ConvRunner(mk, xin.shape, dt, ws, bias, None, A.FLOAT, res_dtype=(dt if with_res else -1),
                     sum_scale=1.0, **kw)
    if expect is not None:
        assert (run.info()["block_n"], run.info()["split"]) == expect, run.info()
    got = run.run(dev(xin), dev(res_in) if with_res else None)
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    max_ratio, max_diff = oracle.tensor_cmp(want, got)
    assert max_diff < 1e-3 or max_ratio <= 1e-3, (max_ratio, max_diff, run.info())
    if math == "tf32x3":
        # the tensor core accumulates in fp32 with truncation: the error grows with the number of accumulation
        # steps (3 MMAs per 8 k-elements), so the bound scales with the reduction length beyond the 1152 of a 3x3x128
        scale_ref = float(np.abs(want).max())
        steps = max(1.0, c * r * r / 1152.0)
        assert max_diff <= 2e-5 * max(1.0, scale_ref) * steps, (max_diff, scale_ref, steps)


# ---------------------------------------------------------------------------------------------------------------
# Slab-staged stride-1 R x S kernel (conv_slab.cu): the tile's input rectangle is staged once per channel chunk
# and the filter taps are row-shifted views of it. Shapes cover every swizzle width (32 / 64 / 128-byte chunks),
# 1 .. 4 channel chunks, all four ResNet feature-map sizes (tiles of 2 x 56, 4 x 28, 7 x 14, 7 x 7 pixels), images
# wider than one tile (tile = part of a row), ragged tile rows, 5 x 5 / non-square filters, no / asymmetric-free
# padding, ragged output channels, and every forced tile width.
# (n, h, w, c, k, r, s, pad_h, pad_w)
SLAB_CASES = [
    (2, 14, 14, 256, 256, 3, 3, 1, 1),
    (8, 7, 7, 512, 512, 3, 3, 1, 1),
    (2, 28, 28, 128, 128, 3, 3, 1, 1),
    (1, 56, 56, 64, 64, 3, 3, 1, 1),
    (1, 12, 12, 32, 48, 3, 3, 1, 1),       # SWIZZLE_32B rows
    (1, 30, 30, 64, 40, 3, 3, 0, 0),       # no padding, ragged channels
    (1, 9, 140, 64, 64, 3, 3, 1, 1),       # wider than a tile: two tiles per row, the second one ragged
    (1, 5, 224, 128, 32, 3, 3, 1, 1),
    (2, 17, 17, 128, 72, 5, 5, 2, 2),      # 5 x 5, ragged tile rows
    (1, 20, 20, 64, 64, 1, 7, 0, 3),       # 1 x 7
    (1, 20, 20, 64, 64, 7, 1, 3, 0),       # 7 x 1
    (3, 10, 10, 384, 96, 3, 3, 2, 2),      # padding wider than the filter needs, 3 chunks
]


def _slab_io(rng, case, in_unsigned):
    n, h, w, c, k, r, s, ph, pw = case
    x = (rng.integers(0, 256, (n, h, w, c)).astype(np.uint8) if in_unsigned
         else rng.integers(-128, 128, (n, h, w, c)).astype(np.int8))
    wq = rng.integers(-127, 128, (k, c, r, s)).astype(np.int8)
    bias = rng.uniform(-2000, 2000, k).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, k).astype(np.float32) * np.float32(1.0 / (40.0 * np.sqrt(c * r * s) * 8))
    return x, wq, bias, scale


@pytest.mark.parametrize("case", SLAB_CASES)
@pytest.mark.parametrize("variant", ["s8_relu_u8", "u8_res_s8", "s8_f32"])
@pytest.mark.parametrize("bn", [0, 32, 64, 128, 256])
def test_conv_slab_int8_bit_exact(case, variant, bn, oracle, monkeypatch):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev, pad_channels
    monkeypatch.setenv("B200_SABER_SLAB", "2")     # run the slab kernel wherever it applies, whatever the estimate says
    if bn:
        if SLAB_CASES.index(case) % 3 != (bn // 64) % 3:
            pytest.skip("forced tile widths are sampled over the shape list")
        monkeypatch.setenv("B200_SABER_FORCE_BN", str(bn))
    rng = np.random.default_rng(hash((case, variant)) % (2 ** 31))
    n, h, w, c, k, r, s, ph, pw = case
    in_unsigned = variant == "u8_res_s8"
    x, wq, bias, scale = _slab_io(rng, case, in_unsigned)
    out_dtype = {"s8_relu_u8": A.UINT8, "u8_res_s8": A.INT8, "s8_f32": A.FLOAT}[variant]
    if out_dtype == A.FLOAT and bn > 128:
        pytest.skip("4-byte outputs cap the tile at 128 channels")
    kw = dict(stride=(1, 1), pad=(ph, pw), dil=(1, 1), relu=variant != "s8_f32")
    res, sum_scale = None, 1.0
    oh, ow = h + 2 * ph - r + 1, w + 2 * pw - s + 1
    if variant == "u8_res_s8":
        res = rng.integers(0, 256, (n, oh, ow, k)).astype(np.uint8)
        sum_scale = 0.37
    want = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, residual=res, sum_scale=sum_scale, out_dtype=out_dtype, **kw)
    ldc = (k + 15) // 16 * 16 if out_dtype != A.FLOAT else (k + 3) // 4 * 4
    run = ConvRunner(A.MATH_I8, x.shape, A.UINT8 if in_unsigned else A.INT8, wq, bias, scale,
                     out_dtype, res_dtype=(A.UINT8 if res is not None else -1), sum_scale=sum_scale, ldc=ldc, **kw)
    info = run.info()
    assert info["slab"], info
    if bn:
        assert info["block_n"] == bn, info
    got = run.run(dev(x), dev(pad_channels(res, ldc)) if res is not None else None)
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    assert (got[..., k:] == 0).all(), "padding channels must stay untouched"
    assert got[..., :k].shape == want.shape
    bad = np.argwhere(got[..., :k] != want)
    assert bad.shape[0] == 0, "%d mismatches, first %s (info %s)" % (bad.shape[0], bad[:5], info)
    # the same plan again into the same buffers (graph replays re-run plans): still exact
    got2 = run.run(dev(x), dev(pad_channels(res, ldc)) if res is not None else None)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got2.cpu().numpy()[..., :k], want)


@pytest.mark.parametrize("case", [(2, 14, 14, 64, 64, 3, 3, 1, 1), (1, 28, 28, 128, 96, 3, 3, 1, 1),
                                  (1, 6, 150, 32, 32, 3, 3, 1, 1), (2, 9, 9, 256, 128, 5, 5, 2, 2),
                                  (1, 40, 224, 64, 64, 3, 3, 1, 1)])
@pytest.mark.parametrize("math", ["f16", "tf32x3"])
@pytest.mark.parametrize("with_res", [False, True])
def test_conv_slab_float(case, math, with_res, oracle, monkeypatch):
    monkeypatch.setenv("B200_SABER_SLAB", "2")
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev
    rng = np.random.default_rng(hash((case, math, with_res)) % (2 ** 31))
    n, h, w, c, k, r, s, ph, pw = case
    x = rng.uniform(-1, 1, (n, h, w, c)).astype(np.float32)
    wt = (rng.standard_normal((k, c, r, s)) * np.sqrt(2.0 / (c * r * s))).astype(np.float32)
    bias = rng.uniform(-0.5, 0.5, k).astype(np.float32)
    kw = dict(stride=(1, 1), pad=(ph, pw), dil=(1, 1), relu=True, neg_slope=0.1)
    oh, ow = h + 2 * ph - r + 1, w + 2 * pw - s + 1
    res = rng.uniform(-1, 1, (n, oh, ow, k)).astype(np.float32) if with_res else None
    if math == "f16":
        xs, ws = x.astype(np.float16), wt.astype(np.float16)
        x_seen, w_seen = xs.astype(np.float32), ws.astype(np.float32)
        mk, dt = A.MATH_F16, A.HALF
        res_in = res.astype(np.float16) if with_res else None
        res_seen = res_in.astype(np.float32) if with_res else None
    else:
        xs, ws = x, wt                       # error-compensated split: exact-fp32 operands, fp32-grade tolerance
        x_seen, w_seen = x, wt
        mk, dt = A.MATH_TF32X3, A.FLOAT
        res_in = res_seen = res
    want = oracle.conv_f32_nhwc(x_seen, w_seen, bias, residual=res_seen, beta=1.0, **kw)
    run = ConvRunner(mk, xs.shape, dt, ws, bias, None, A.FLOAT, res_dtype=(dt if with_res else -1), sum_scale=1.0, **kw)
    assert run.info()["slab"], run.info()
    got = run.run(dev(xs), dev(res_in) if with_res else None)
    torch.cuda.synchronize()
    max_ratio, max_diff = oracle.tensor_cmp(want, got.cpu().numpy())
    assert max_diff < 1e-3 or max_ratio <= 1e-3, (max_ratio, max_diff, run.info())
    if math == "tf32x3":
        # the tensor core accumulates in fp32 with truncation: the error grows with the number of accumulation
        # steps (3 MMAs per 8 k-elements), so the bound scales with the reduction length beyond the 1152 of a 3x3x128
        scale_ref = float(np.abs(want).max())
        steps = max(1.0, c * r * s / 1152.0)
        assert max_diff <= 2e-5 * max(1.0, scale_ref) * steps, (max_diff, scale_ref, steps)


# ---------------------------------------------------------------------------------------------------------------
# Persistent tile-pipelined kernel (conv_persistent.cu): one CTA per SM walks the tile list with register accumulators.
# Forced on (B200_SABER_PERSISTENT=2) so that small grids exercise it too: CTAs with 1, 2 and many tiles, several
# n-tiles (bias / scale tables reloaded mid-walk), residual buffer hand-back, ragged last m-tile, strided and 3x3 im2col.
# (n, h, w, c, k, r, stride, pad)
PERSISTENT_CASES = [
    (8, 56, 56, 64, 256, 1, 1, 0),      # 196 tiles on 132 CTAs
    (32, 56, 56, 64, 64, 1, 1, 0),      # 784 tiles: 5-6 per CTA
    (4, 28, 28, 128, 512, 1, 1, 0),     # several n-tiles per CTA walk
    (6, 30, 30, 32, 72, 3, 2, 1),       # strided 3x3, ragged channels and rows
    (2, 9, 9, 256, 40, 1, 1, 0),        # fewer tiles than SMs
    (16, 28, 28, 256, 128, 1, 2, 0),
]


@pytest.mark.parametrize("case", PERSISTENT_CASES)
@pytest.mark.parametrize("variant", ["s8_relu_u8", "u8_res_s8", "s8_f32"])
def test_conv_persistent_int8_bit_exact(case, variant, oracle, monkeypatch):
    monkeypatch.setenv("B200_SABER_PERSISTENT", "2")
    monkeypatch.setenv("B200_SABER_SLAB", "0")
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev, pad_channels
    rng = np.random.default_rng(hash((case, variant)) % (2 ** 31))
    n, h, w, c, k, r, stride, pad = case
    in_unsigned = variant == "u8_res_s8"
    x, wq, bias, scale = _slab_io(rng, (n, h, w, c, k, r, r, pad, pad), in_unsigned)
    out_dtype = {"s8_relu_u8": A.UINT8, "u8_res_s8": A.INT8, "s8_f32": A.FLOAT}[variant]
    kw = dict(stride=(stride, stride), pad=(pad, pad), dil=(1, 1), relu=variant != "s8_f32")
    res, sum_scale = None, 1.0
    oh = oracle.conv_out_size(h, pad, 1, r, stride)
    ow = oracle.conv_out_size(w, pad, 1, r, stride)
    if variant == "u8_res_s8":
        res = rng.integers(0, 256, (n, oh, ow, k)).astype(np.uint8)
        sum_scale = 0.37
    want = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, residual=res, sum_scale=sum_scale, out_dtype=out_dtype, **kw)
    ldc = (k + 15) // 16 * 16 if out_dtype != A.FLOAT else (k + 3) // 4 * 4
    run = ConvRunner(A.MATH_I8, x.shape, A.UINT8 if in_unsigned else A.INT8, wq, bias, scale,
                     out_dtype, res_dtype=(A.UINT8 if res is not None else -1), sum_scale=sum_scale, ldc=ldc, **kw)
    info = run.info()
    assert info["persistent"] and not info["slab"], info
    for rep in range(2):
        got = run.run(dev(x), dev(pad_channels(res, ldc)) if res is not None else None)
        torch.cuda.synchronize()
        got = got.cpu().numpy()
        assert (got[..., k:] == 0).all(), "padding channels must stay untouched"
        bad = np.argwhere(got[..., :k] != want)
        assert bad.shape[0] == 0, "%d mismatches, first %s (info %s)" % (bad.shape[0], bad[:5], info)


@pytest.mark.parametrize("math", ["f16"])
def test_conv_persistent_float(math, oracle, monkeypatch):
    monkeypatch.setenv("B200_SABER_PERSISTENT", "2")
    monkeypatch.setenv("B200_SABER_SLAB", "0")
    test_conv_float((2, 28, 28, 128, 128, 3, 1, 1, 1), math, True, oracle)
    test_conv_float((2, 24, 24, 64, 64, 1, 1, 0, 1), math, False, oracle)


# ---------------------------------------------------------------------------------------------------------------
# Fused MAX pooling in the conv plan's epilogue (b200_conv_desc_t::fuse_pool; SaberConv2DPooling,
# saber_conv_pooling.cpp:36-130): bit-exact against conv -> pool of the oracle (int8), reference criterion (float).
# (n, h, w, c, k, r, pad, pool window, pool stride, pool pad)
POOL_CASES = [
    (2, 56, 56, 64, 64, 3, 1, 2, 2, 0),       # VGG-style 3x3 + 2x2/s2
    (1, 224, 224, 64, 64, 3, 1, 2, 2, 0),     # VGG16 conv1_2 + pool1 at full size
    (2, 28, 28, 128, 256, 3, 1, 2, 2, 0),     # several n-tiles
    (1, 30, 26, 32, 48, 3, 1, 3, 2, 0),       # overlapping window (3x3/s2), ceil-mode ragged edge, k = 48
    (1, 14, 14, 512, 512, 3, 1, 2, 2, 0),     # VGG16 conv5_3 + pool5
    (2, 17, 19, 64, 32, 5, 2, 3, 2, 1),       # 5x5 filter, padded pooling window
    (1, 12, 12, 64, 64, 3, 0, 2, 1, 0),       # stride-1 pooling
]


@pytest.mark.parametrize("case", POOL_CASES)
@pytest.mark.parametrize("variant", ["u8", "s8"])
def test_conv_fused_pool_int8_bit_exact(case, variant, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev
    rng = np.random.default_rng(abs(hash((case, variant))) % (2 ** 31))
    n, h, w, c, k, r, pad, pk, ps, pp = case
    x = rng.integers(0, 256, (n, h, w, c)).astype(np.uint8)
    wq = rng.integers(-127, 128, (k, c, r, r)).astype(np.int8)
    bias = rng.uniform(-2000, 2000, k).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, k).astype(np.float32) * np.float32(1.0 / (40.0 * np.sqrt(c * r * r) * 8))
    out_dtype = A.UINT8 if variant == "u8" else A.INT8
    relu = variant == "u8"
    conv = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, out_dtype=out_dtype, pad=(pad, pad), relu=relu)
    want = oracle.pool_s8_nhwc(conv, (pk, pk), (pp, pp), (ps, ps), A.POOL_MAX)
    ldc = (k + 15) // 16 * 16
    run = ConvRunner(A.MATH_I8, x.shape, A.UINT8, wq, bias, scale, out_dtype, pad=(pad, pad), relu=relu, ldc=ldc,
                     fuse_pool=pk, pool_stride=ps, pool_pad=pp)
    assert run.info()["slab"]
    got = run.run(dev(x))
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    assert (got[..., k:] == 0).all()
    assert got[..., :k].shape == want.shape, (got.shape, want.shape)
    np.testing.assert_array_equal(got[..., :k], want)


@pytest.mark.parametrize("case", [POOL_CASES[0], POOL_CASES[3], POOL_CASES[4]])
@pytest.mark.parametrize("math", ["f16", "tf32x3"])
def test_conv_fused_pool_float(case, math, oracle):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev
    rng = np.random.default_rng(abs(hash((case, math))) % (2 ** 31))
    n, h, w, c, k, r, pad, pk, ps, pp = case
    x = rng.uniform(-1, 1, (n, h, w, c)).astype(np.float32)
    wt = (rng.standard_normal((k, c, r, r)) * np.sqrt(2.0 / (c * r * r))).astype(np.float32)
    bias = rng.uniform(-0.5, 0.5, k).astype(np.float32)
    if math == "f16":
        xs, ws = x.astype(np.float16), wt.astype(np.float16)
        x_seen, w_seen, mk, dt = xs.astype(np.float32), ws.astype(np.float32), A.MATH_F16, A.HALF
    else:
        xs, ws, x_seen, w_seen, mk, dt = x, wt, x, wt, A.MATH_TF32X3, A.FLOAT
    conv = oracle.conv_f32_nhwc(x_seen, w_seen, bias, pad=(pad, pad), relu=True, neg_slope=0.1)
    want = oracle.pool_f32(conv, (pk, pk), (pp, pp), (ps, ps), A.POOL_MAX, nhwc=True)
    run = ConvRunner(mk, xs.shape, dt, ws, bias, None, A.FLOAT, pad=(pad, pad), relu=True, neg_slope=0.1,
                     fuse_pool=pk, pool_stride=ps, pool_pad=pp)
    got = run.run(dev(xs))
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    assert got.shape == want.shape, (got.shape, want.shape)
    max_ratio, max_diff = oracle.tensor_cmp(want, got)
    assert max_diff < 1e-3 or max_ratio <= 1e-3, (max_ratio, max_diff, run.info())


def test_conv_fused_pool_rejects_what_it_cannot_fuse():
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner
    wq = np.ones((64, 64, 1, 1), np.int8)
    with pytest.raises(A.SaberError):     # 1x1 conv: no rectangle tiling -> UNIMPL, the caller pools separately
        ConvRunner(A.MATH_I8, (1, 8, 8, 64), A.UINT8, wq, None, None, A.UINT8, fuse_pool=2, pool_stride=2)
