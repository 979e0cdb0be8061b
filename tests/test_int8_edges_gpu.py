"""GPU: the INT8 kernels at their numeric edges, bit for bit against the CPU oracle.

Random data under moderate scales never reaches the places where an 8-bit kernel can be subtly wrong, so every case
here is designed data:
- rounding ties of both signs and both parities, under the three rules the kernels use: round half to even (conv, fc,
  depthwise and head epilogues, pooling averages), round half away from zero (eltwise sum, s8 graph-input
  quantisation) and truncation (u8 graph-input quantisation);
- both clamp bounds of every 8-bit output, with and without relu;
- s32 accumulators past 2^24, where the conversion to fp32 rounds, through every split-K factor and kernel;
- pooling windows of 255..272 taps over saturated planes, around the exact range of packed 16-bit sums.

The expected results always come from the oracle (oracle/oracle.c). Every generator also asserts its own coverage on
the oracle's pre-rounding values, so an edit that makes a case vacuous fails that case.
"""
import ctypes as C
import functools

import numpy as np
import pytest

from anakin_b200 import saber_abi as A

pytestmark = pytest.mark.gpu

_TDT = {A.INT8: "int8", A.UINT8: "uint8", A.FLOAT: "float32"}
_BOUNDS = {A.INT8: (-128, 127), A.UINT8: (0, 255)}
_DT = {"s8": A.INT8, "u8": A.UINT8, "f32": A.FLOAT}


def _torch_dt(dt):
    import torch
    return getattr(torch, _TDT[dt])


def _out_range(out_dtype, relu):
    lo, hi = _BOUNDS[out_dtype]
    return (max(lo, 0) if relu else lo), hi


def _tie_classes(pre, lo, hi):
    """{(sign, parity of the integer part): count} of the exact half-integers among `pre` that round into [lo, hi]."""
    v = np.asarray(pre, np.float64).ravel()
    t = v[(np.abs(v - np.trunc(v)) == 0.5) & (v > lo - 0.5) & (v < hi + 0.5)]
    k = np.trunc(np.abs(t)).astype(np.int64) % 2
    return {(s, p): int(((np.sign(t) == s) & (k == p)).sum()) for s in (-1, 1) for p in (0, 1)}


def assert_ties(pre, lo, hi, at_least=20, what=""):
    """Ties of both parities; negative ones too where the output range and the data both reach below -1."""
    got = _tie_classes(pre, lo, hi)
    negative = lo < 0 and (np.asarray(pre) < -1).any()
    for (s, p), n in got.items():
        if s < 0 and not negative:
            continue
        assert n >= at_least, "too few ties of sign %d, parity %d in %s: %s" % (s, p, what, got)


def assert_clamps(pre, lo, hi, what=""):
    """Pre-rounding values beyond both clamp bounds (the lower one is relu's 0 where relu folds into the clamp)."""
    v = np.asarray(pre, np.float64)
    assert (v < lo - 0.5).any() and (v > hi + 0.5).any(), "%s must saturate at both %d and %d" % (what, lo, hi)


def roundf(v):
    """C roundf (half away from zero) of fp32 values, exactly."""
    v = np.asarray(v, np.float64)
    return np.sign(v) * np.floor(np.abs(v) + 0.5)


def _dev_out(shape, dt, fill=0):
    import torch
    return torch.full(shape, fill, dtype=_torch_dt(dt), device="cuda")


# ================================================================================ a. conv epilogue grid
# A 1x1 conv (or the centre tap of a padded 3x3) whose accumulator is x0 + 127 * x1: input channels 0 and 1 carry x0
# and x1, their weights are 1 and 127, everything else is zero. The 65536 pixels hold every (x0, x1) pair, so the
# accumulator sweeps [-16384, 16256] for s8 inputs and [0, 32640] for u8. The output channels are a table of
# (bias, scale) pairs: power-of-two scales with integer and half-integer biases (ties of both signs and parities),
# scales that saturate both ends, and inexact scales (near-ties).
GRID_H, GRID_W, GRID_C = 128, 512, 32


def grid_pairs():
    pow2 = [2.0 ** -e for e in range(9)]
    inexact = [0.1, 1 / 3, 0.7, 0.013]
    biases = [0.0, 0.5, -0.5, 1.0, -1.0, 2.5, -3.5, 64.0, -64.5, 127.5, -1000.0, 4000.5, -8000.0, 16000.0, -16384.5]
    pairs = [(b, s) for s in pow2 + inexact for b in biases]
    pairs += [(0.5, 2.0), (-0.5, 2.0), (0.0, 4.0), (0.25, 2.0), (0.0, 1e-3), (-0.25, 0.5), (7.0, 0.125), (-7.0, 0.125),
              (0.75, 0.25), (-0.75, 0.25), (0.0, 0.0), (1.5, 1.0), (-1.5, 1.0)]
    b, s = np.array(pairs, np.float64).T
    return b.astype(np.float32), s.astype(np.float32)


def grid_input(unsigned):
    p = np.arange(GRID_H * GRID_W)
    lo = 0 if unsigned else -128
    x = np.zeros((1, GRID_H, GRID_W, GRID_C), np.int16)
    x[0, ..., 0] = (p % 256 + lo).reshape(GRID_H, GRID_W)
    x[0, ..., 1] = (p // 256 + lo).reshape(GRID_H, GRID_W)
    return x.astype(np.uint8 if unsigned else np.int8)


def grid_weights(k, r):
    w = np.zeros((k, GRID_C, r, r), np.int8)
    w[:, 0, r // 2, r // 2] = 1
    w[:, 1, r // 2, r // 2] = 127
    return w


def grid_residual(k, dtype):
    """Every residual code at every channel, in a pattern that differs between neighbouring pixels and channels."""
    p = np.arange(GRID_H * GRID_W)[:, None]
    j = np.arange(k)[None, :]
    r = (p * 5 + j * 3) % 256 - (128 if dtype == A.INT8 else 0)
    return r.reshape(1, GRID_H, GRID_W, k).astype(np.int8 if dtype == A.INT8 else np.uint8)


# name: (input unsigned, output, relu, residual dtype, sum_scale)
GRID_VARIANTS = {
    "s8_s8": (False, A.INT8, False, None, 1.0),
    "s8_relu_u8": (False, A.UINT8, True, None, 1.0),
    "u8_u8": (True, A.UINT8, False, None, 1.0),
    "u8_relu_s8": (True, A.INT8, True, None, 1.0),
    "u8_f32": (True, A.FLOAT, False, None, 1.0),
    "s8_relu_f32": (False, A.FLOAT, True, None, 1.0),
    "u8_res-s8-1_s8": (True, A.INT8, False, A.INT8, 1.0),
    "s8_res-u8-0.5_relu_u8": (False, A.UINT8, True, A.UINT8, 0.5),
    "s8_res-s8-0.5_relu_s8": (False, A.INT8, True, A.INT8, 0.5),
    "u8_res-u8-0.37_s8": (True, A.INT8, False, A.UINT8, 0.37),
    "s8_res-s8-0.37_u8": (False, A.UINT8, False, A.INT8, 0.37),
}


@functools.lru_cache(maxsize=None)
def grid_case(variant, k):
    """(x, bias, scale, residual, expected output) of one grid variant, after checking its coverage. The 1x1 design and
    the centre tap of the padded 3x3 have the same accumulators, so one oracle result serves both."""
    from oracle import pyoracle as oracle
    unsigned, out_dtype, relu, res_dtype, sum_scale = GRID_VARIANTS[variant]
    x = grid_input(unsigned)
    bias, scale = (a[:k] for a in grid_pairs())
    w = grid_weights(k, 1)
    res = grid_residual(k, res_dtype) if res_dtype is not None else None
    kw = dict(residual=res, sum_scale=sum_scale)
    want = oracle.conv_s8_nhwc_x86(x, w, bias, scale, out_dtype=out_dtype, relu=relu, **kw)
    pre = oracle.conv_s8_nhwc_x86(x, w, bias, scale, out_dtype=A.FLOAT, relu=False, **kw)
    acc = oracle.conv_s8_nhwc_x86(x, w, None, None, out_dtype=A.FLOAT)
    assert acc.min() == (0 if unsigned else -16384) and acc.max() == (32640 if unsigned else 16256)
    if out_dtype != A.FLOAT:
        lo, hi = _out_range(out_dtype, relu)
        assert_clamps(pre, lo, hi, variant)
        assert (want == lo).any() and (want == hi).any(), variant
        if sum_scale in (1.0, 0.5):
            assert_ties(pre, lo, hi, what=variant)
        else:
            # an inexact sum_scale: the oracle's fmaf and a separate multiply and add round some values differently
            f = oracle.conv_s8_nhwc_x86(x, w, bias, scale, out_dtype=A.FLOAT)
            unfused = np.float32(res.astype(np.float32) * np.float32(sum_scale)) + f
            sep = (np.rint(unfused) != np.rint(pre)) & (pre > lo - 0.5) & (pre < hi + 0.5)
            assert sep.sum() >= 5, "%s: no value separates fused from unfused arithmetic" % variant
    else:
        assert (pre < 0).any() and (pre > 0).any() and (pre != np.rint(pre)).any()
    return x, bias, scale, res, want


def _ldc(k, out_dtype):
    return (k + 15) // 16 * 16 if out_dtype != A.FLOAT else (k + 3) // 4 * 4


def run_conv(x, w, bias, scale, out_dtype, relu, res=None, res_dtype=None, sum_scale=1.0, pad=0, **kw):
    """One conv plan on designed data: (output without the padding channels, plan info)."""
    import torch
    from gpu_util import ConvRunner, dev, pad_channels
    k = w.shape[0]
    ldc = _ldc(k, out_dtype)
    run = ConvRunner(A.MATH_I8, x.shape, A.UINT8 if x.dtype == np.uint8 else A.INT8, w, bias, scale, out_dtype,
                     res_dtype=res_dtype if res is not None else -1, sum_scale=sum_scale, ldc=ldc, pad=(pad, pad),
                     relu=relu, **kw)
    info = run.info()
    got = run.run(dev(x), dev(pad_channels(res, ldc)) if res is not None else None)
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    assert (got[..., k:] == 0).all(), "padding channels must stay untouched"
    return got[..., :k], info


GRID_KERNELS = ["tile32", "tile64", "tile128", "tile256", "slab", "persistent"]


@pytest.mark.parametrize("kernel", GRID_KERNELS)
@pytest.mark.parametrize("variant", list(GRID_VARIANTS))
def test_conv_epilogue_grid(variant, kernel, monkeypatch):
    unsigned, out_dtype, relu, res_dtype, sum_scale = GRID_VARIANTS[variant]
    k = 200     # ragged against every tile width
    x, bias, scale, res, want = grid_case(variant, k)
    r, pad = 1, 0
    if kernel.startswith("tile"):
        bn = int(kernel[4:])
        if out_dtype == A.FLOAT and bn > 128:
            pytest.skip("4-byte outputs cap the tile at 128 channels")
        monkeypatch.setenv("B200_SABER_FORCE_BN", str(bn))
        monkeypatch.setenv("B200_SABER_PERSISTENT", "0")
    elif kernel == "slab":
        monkeypatch.setenv("B200_SABER_SLAB", "2")
        r, pad = 3, 1
    else:
        monkeypatch.setenv("B200_SABER_PERSISTENT", "2")
        monkeypatch.setenv("B200_SABER_SLAB", "0")
        monkeypatch.setenv("B200_SABER_FORCE_SPLIT", "1")     # the persistent kernel takes unsplit plans only
    got, info = run_conv(x, grid_weights(k, r), bias, scale, out_dtype, relu, res, res_dtype, sum_scale, pad)
    if kernel.startswith("tile"):
        assert info["block_n"] == bn and not info["slab"] and not info["persistent"], info
    else:
        assert info[kernel], info
    bad = np.argwhere(got != want)
    assert bad.shape[0] == 0, "%d mismatches, first %s: got %s want %s (info %s)" % (
        bad.shape[0], bad[:5].tolist(), got[tuple(bad[:5].T)], want[tuple(bad[:5].T)], info)


@pytest.mark.parametrize("pool", [(2, 2, 0), (3, 2, 0)])
@pytest.mark.parametrize("variant", ["s8_s8", "s8_relu_u8", "u8_u8"])
def test_conv_epilogue_grid_fused_max_pool(variant, pool, oracle):
    """The slab kernel with its fused MAX pooling: the requantised grid, then the window maxima."""
    unsigned, out_dtype, relu, _, _ = GRID_VARIANTS[variant]
    k = 208     # a fused pooling needs whole 16-byte output rows
    x, bias, scale, _, conv = grid_case(variant, k)
    want = oracle.pool_s8_nhwc(conv, (pool[0],) * 2, (pool[2],) * 2, (pool[1],) * 2, A.POOL_MAX)
    got, info = run_conv(x, grid_weights(k, 3), bias, scale, out_dtype, relu, pad=1, fuse_pool=pool[0],
                         pool_stride=pool[1], pool_pad=pool[2])
    assert info["slab"], info
    assert got.shape == want.shape, (got.shape, want.shape)
    np.testing.assert_array_equal(got, want)


# ================================================================================ b. accumulators past 2^24
# Saturated inputs (u8 255, or s8 -128 with channel 0 at -127 so that the sums stay odd) against weights of +-127,
# with a few weights per output channel lowered so that each channel's accumulator is a distinct odd value between
# 2^24 and about 2^27 in magnitude, of both signs. fp32 outputs show the acc -> fp32 rounding directly; the 8-bit
# outputs take power-of-two scales that bring the values back into range.
def big_weights(k, kk, unsigned):
    """[k][kk] int8: row j sums to sign_j * (127 * kk - d_j), with the lowering taken from the end of the row."""
    max_sum = 127 * kk
    floor = (2 ** 24) // (255 if unsigned else 128) + 1          # |acc| > 2^24
    step = (max_sum - floor) * 9 // 10 // (2 * k)
    w = np.empty((k, kk), np.int16)
    for j in range(k):
        sign = 1 if j % 2 == 0 else -1
        d = 1 + 2 * j * step
        if unsigned and (max_sum - d) % 2 == 0:      # 255 * S is odd when S is
            d += 1
        row = np.full(kk, 127, np.int16)
        q, rem = divmod(d, 254)
        assert q + 1 < kk - 16, "channel 0's weights must keep their odd +-127"
        row[kk - q:] = -127
        row[kk - q - 1] -= rem
        w[j] = sign * row
    return w.astype(np.int8)


def big_input(shape, unsigned):
    if unsigned:
        return np.full(shape, 255, np.uint8)
    x = np.full(shape, -128, np.int8)
    x[..., 0] = -127
    return x


def exact_acc(x, w_kcrs, pad):
    """The exact accumulators (float64 sums of integer products stay exact at these sizes)."""
    n, h, wd, c = x.shape
    k, _, r, s = w_kcrs.shape
    xp = np.zeros((n, h + 2 * pad, wd + 2 * pad, c), np.float64)
    xp[:, pad:pad + h, pad:pad + wd] = x
    acc = np.zeros((n, h + 2 * pad - r + 1, wd + 2 * pad - s + 1, k), np.float64)
    for ky in range(r):
        for kx in range(s):
            acc += xp[:, ky:ky + acc.shape[1], kx:kx + acc.shape[2]] @ w_kcrs[:, :, ky, kx].astype(np.float64).T
    return acc


def assert_big_acc(acc, centre):
    """Most accumulators past 2^24 and inexact in fp32; at one full-window pixel, distinct odd values of both signs."""
    a = np.abs(acc)
    assert a.max() < 2 ** 31
    big = (a > 2 ** 24) & (acc.astype(np.float32).astype(np.float64) != acc)
    assert big.mean() >= 0.5, "only %.2f of the accumulators are past 2^24 and inexact in fp32" % big.mean()
    assert len(np.unique(centre)) == centre.size and (centre % 2 != 0).all()
    assert (centre > 2 ** 24).any() and (centre < -2 ** 24).any()


# name: (n, h, w, c, r, pad)
BIG_SHAPES = {"1x1_c2048": (1, 12, 12, 2048, 1, 0), "3x3_c512": (1, 14, 14, 512, 3, 1)}


@functools.lru_cache(maxsize=None)
def big_case(shape, unsigned, out):
    from oracle import pyoracle as oracle
    n, h, w, c, r, pad = BIG_SHAPES[shape]
    k = 200
    x = big_input((n, h, w, c), unsigned)
    wq = big_weights(k, c * r * r, unsigned).reshape(k, c, r, r)
    acc = exact_acc(x, wq, pad)
    assert_big_acc(acc, acc[0, h // 2, w // 2])
    out_dtype = _DT[out]
    relu = out_dtype == A.UINT8
    if out_dtype == A.FLOAT:
        bias, scale = None, None
    else:
        top = 7 if out_dtype == A.INT8 else 8
        e = np.ceil(np.log2(np.abs(acc).reshape(-1, k).max(0))) - top
        scale = (2.0 ** -e).astype(np.float32)
        bias = np.where(np.arange(k) % 3 == 0, 0.5, 0.0).astype(np.float32) / scale
    want = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, out_dtype=out_dtype, relu=relu, pad=(pad, pad))
    if out_dtype == A.FLOAT:
        assert (want.astype(np.float64) != acc).mean() >= 0.5
    else:
        lo, hi = _out_range(out_dtype, relu)
        assert ((want > lo) & (want < hi)).mean() >= 0.3, "the scales must keep most values in range"
    return x, wq, bias, scale, relu, pad, want


BIG_KERNELS = {"split1": (64, 1), "split2": (32, 2), "split4": (64, 4), "split8": (128, 8), "slab": None,
               "persistent": None}


@pytest.mark.parametrize("out", ["f32", "s8", "u8"])
@pytest.mark.parametrize("unsigned", [True, False], ids=["u8in", "s8in"])
@pytest.mark.parametrize("kernel", list(BIG_KERNELS))
@pytest.mark.parametrize("shape", list(BIG_SHAPES))
def test_conv_large_accumulators(shape, kernel, unsigned, out, monkeypatch):
    if kernel == "slab" and shape.startswith("1x1"):
        pytest.skip("the slab kernel runs R x S filters only")
    x, wq, bias, scale, relu, pad, want = big_case(shape, unsigned, out)
    if kernel.startswith("split"):
        bn, split = BIG_KERNELS[kernel]
        monkeypatch.setenv("B200_SABER_FORCE_BN", str(bn))
        monkeypatch.setenv("B200_SABER_FORCE_SPLIT", str(split))
        monkeypatch.setenv("B200_SABER_SLAB", "0")
        monkeypatch.setenv("B200_SABER_PERSISTENT", "0")
    elif kernel == "slab":
        monkeypatch.setenv("B200_SABER_SLAB", "2")
    else:
        monkeypatch.setenv("B200_SABER_PERSISTENT", "2")
        monkeypatch.setenv("B200_SABER_SLAB", "0")
        monkeypatch.setenv("B200_SABER_FORCE_SPLIT", "1")     # the persistent kernel takes unsplit plans only
    got, info = run_conv(x, wq, bias, scale, _DT[out], relu, pad=pad)
    if kernel.startswith("split"):
        assert (info["block_n"], info["split"]) == (bn, split) and not info["slab"] and not info["persistent"], info
    else:
        assert info[kernel], info
    np.testing.assert_array_equal(got, want)


def _fc_desc(m, k, n, in_dtype, out_dtype, relu=False):
    d = A.FcStreamDesc()
    d.math, d.in_dtype, d.out_dtype = A.MATH_I8, in_dtype, out_dtype
    d.m, d.k, d.ldx, d.n_out = m, k, k, n
    d.ldo = (n + 15) // 16 * 16
    d.relu = int(relu)
    return d


def run_fc(x, w, bias, scale, out_dtype, relu=False):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    m, k = x.shape
    n = w.shape[0]
    lib = A.load()
    assert m <= lib.b200_fc_stream_max_rows()
    d = _fc_desc(m, k, n, A.UINT8 if x.dtype == np.uint8 else A.INT8, out_dtype, relu)
    out = _dev_out((m, d.ldo), out_dtype)
    xd, wd, bd, sd = dev(x), dev(w), dev(bias), dev(scale)     # alive until the kernel has run
    A.check(lib.b200_fc_stream_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), ptr(sd), ptr(out), stream_ptr()), "fc_stream")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert (got[:, n:] == 0).all()
    return got[:, :n]


@functools.lru_cache(maxsize=None)
def big_fc_case(k, n):
    """u8 rows of 255 against the big_weights design: odd, distinct accumulators past 2^24 (up to 8e8 at k = 25088)."""
    from oracle import pyoracle as oracle
    x = np.full((8, 1, 1, k), 255, np.uint8)
    w = big_weights(n, k, True)
    acc = x[:1, 0, 0].astype(np.float64) @ w.astype(np.float64).T
    assert_big_acc(acc, acc[0])
    zeros, ones = np.zeros(n, np.float32), np.ones(n, np.float32)
    want = oracle.conv_s8_nhwc_x86(x, w.reshape(n, k, 1, 1), zeros, ones, out_dtype=A.FLOAT).reshape(8, n)
    return x.reshape(8, k), w, zeros, ones, want


@pytest.mark.parametrize("m", range(1, 9))
def test_fc_stream_large_accumulators(m):
    """VGG's fc6 reduction length: accumulators up to 8e8."""
    x, w, zeros, ones, want = big_fc_case(25088, 200)
    np.testing.assert_array_equal(run_fc(x[:m], w, zeros, ones, A.FLOAT), want[:m])


@pytest.mark.parametrize("pool_max", [0, 1], ids=["avg", "max"])
@pytest.mark.parametrize("m", range(1, 9))
def test_head_large_accumulators(m, pool_max):
    """The fused head at c = 2048 on saturated planes: pooled codes of 255, fp32 logits of accumulators past 2^24."""
    x, w, zeros, ones, want = big_fc_case(2048, 200)
    planes = np.full((m, 7, 7, 2048), 255, np.uint8)
    pooled, logits = run_head(planes, w, zeros, ones, pool_max)
    assert (pooled == 255).all()
    np.testing.assert_array_equal(logits, want[:m])


def run_head(x, w, bias, scale, pool_max, expect=A.SUCCESS):
    """b200_head_run on NHWC planes [m][h][w][c]: (pooled codes, fp32 logits), or None when it must refuse."""
    import torch
    from gpu_util import dev, ptr, stream_ptr
    lib = A.load()
    m, h, wd, c = x.shape
    n = w.shape[0]
    in_dtype = A.UINT8 if x.dtype == np.uint8 else A.INT8
    hd = A.HeadDesc()
    hd.fc, hd.hw, hd.pool_max = _fc_desc(m, c, n, in_dtype, A.FLOAT), h * wd, pool_max
    hd.ldp = hd.fc.ldo
    pooled = _dev_out((m, c), in_dtype)
    logits = _dev_out((m, hd.fc.ldo), A.FLOAT)
    prob = _dev_out((m, hd.ldp), A.FLOAT)
    ws = _dev_out((lib.b200_head_workspace_bytes(C.byref(hd)),), A.UINT8)
    xd, wd, bd, sd = dev(x), dev(w), dev(bias), dev(scale)     # alive until the kernel has run
    st = lib.b200_head_run(C.byref(hd), ptr(xd), ptr(pooled), ptr(wd), ptr(bd), ptr(sd), ptr(logits), ptr(prob), ptr(ws),
                           stream_ptr())
    assert st == expect, (st, expect)
    if st != A.SUCCESS:
        return None
    torch.cuda.synchronize()
    return pooled.cpu().numpy(), logits.cpu().numpy()[:, :n]


# ================================================================================ c. graph-input quantisation ties
IN_SHIFT = 5                          # input scale 2^-5: quantisation multiplies by 32, exactly


def tie_values(unsigned):
    """fp32 inputs on the half steps (k + 0.5) * s of the quantisation grid, +-1 ulp around them, past both clamp
    bounds, and +-0.0. u8 quantisation truncates x / (s * 127/255), so its values sit on that grid's half steps."""
    s = np.float32(2.0 ** -IN_SHIFT)
    if unsigned:
        inv = np.float32(1) / (s * (np.float32(127) / np.float32(255)))
        k = np.arange(-6, 266)
        t = ((k + 0.5) / inv).astype(np.float32)
    else:
        k = np.arange(-140, 141)
        t = ((k + 0.5) * s).astype(np.float32)
    v = np.concatenate([t, np.nextafter(t, np.float32(np.inf)), np.nextafter(t, np.float32(-np.inf)),
                        np.array([0.0, -0.0, 1e6, -1e6, 200 * s, -200 * s], np.float32)])
    return v.astype(np.float32), s


def tie_tensor(shape, unsigned):
    v, s = tie_values(unsigned)
    x = np.resize(v, int(np.prod(shape))).reshape(shape).astype(np.float32)
    assert np.signbit(x[x == 0]).any(), "-0.0 must be among the inputs"
    return x, s


def assert_input_ties(x, s, unsigned):
    t = np.asarray(x, np.float32).astype(np.float64) * 2.0 ** IN_SHIFT
    if unsigned:
        t = t * (255.0 / 127.0)
        frac = t - np.floor(t)
        assert ((frac > 0.4) & (frac < 0.6) & (t > 0) & (t < 255)).sum() >= 200
        assert (t > 256).any() and (t < 0).any()
    else:
        assert_ties(t, -128, 127, what="the quantised inputs")
        assert_clamps(t, -128, 127, "the quantised inputs")


@pytest.mark.parametrize("c", [3, 40], ids=["c3-pixel-kernel", "c40-transpose-kernel"])
@pytest.mark.parametrize("out", ["s8", "u8"])
def test_nchw_to_nhwc_quantisation_ties(c, out, oracle):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    unsigned = out == "u8"
    n, h, w = 2, 19, 23
    x, s = tie_tensor((n, c, h, w), unsigned)
    assert_input_ties(x, s, unsigned)
    xt = np.ascontiguousarray(x.transpose(0, 2, 3, 1))
    want = oracle.quant_fp32_u8(xt, s) if unsigned else oracle.quant_fp32_s8(xt, s)
    inv = np.float32(1) / (s * (np.float32(127) / np.float32(255))) if unsigned else np.float32(1) / s
    c_pad = (c + 15) // 16 * 16
    got = _dev_out((n, h, w, c_pad), _DT[out], 77)
    xd = dev(x)
    A.check(A.load().b200_nchw_to_nhwc(ptr(xd), ptr(got), _DT[out], n, c, h, w, c_pad, float(inv), stream_ptr()))
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    np.testing.assert_array_equal(got[..., :c], want)
    assert (got[..., c:] == 0).all()


STEM_TIE_CASES = [(2, 3, 40, 44, 64, 7, 7, 2, 3, (3, 2, 0)), (1, 3, 33, 35, 32, 3, 3, 1, 1, None)]


@pytest.mark.parametrize("monotone", [0, 1])
@pytest.mark.parametrize("out", ["f32", "relu_u8", "s8"])
@pytest.mark.parametrize("case", STEM_TIE_CASES, ids=["7x7s2-pool", "3x3s1"])
def test_stem_conv_quantisation_ties(case, out, monotone, oracle):
    """The stem's in-kernel quantisation of tie inputs; fp32 outputs show any differing code directly."""
    from test_stem_gpu import _run_stem, _stem_desc
    n, c, h, w, k, r, s_, stride, pad, pool = case
    if monotone and pool is None:
        pytest.skip("the flag only matters with a fused pooling")
    x, s = tie_tensor((n, c, h, w), False)
    assert_input_ties(x, s, False)
    wq = np.random.default_rng(17).integers(-127, 128, (k, c, r, s_)).astype(np.int8)
    out_dtype = {"f32": A.FLOAT, "relu_u8": A.UINT8, "s8": A.INT8}[out]
    relu = out == "relu_u8"
    if out_dtype == A.FLOAT:
        bias, scale = np.zeros(k, np.float32), np.ones(k, np.float32)
    else:
        bias = np.zeros(k, np.float32)
        scale = np.full(k, 1.0 / (40.0 * np.sqrt(c * r * s_) * 8), np.float32)
    xq = oracle.quant_fp32_s8(np.ascontiguousarray(x.transpose(0, 2, 3, 1)), s)
    want = oracle.conv_s8_nhwc_x86(xq, wq, bias, scale, out_dtype=out_dtype, stride=(stride, stride), pad=(pad, pad),
                                   relu=relu)
    if pool is not None:
        pk = ((pool[0],) * 2, (pool[2],) * 2, (pool[1],) * 2)
        want = (oracle.pool_f32(want, *pk, A.POOL_MAX, nhwc=True) if out_dtype == A.FLOAT
                else oracle.pool_s8_nhwc(want, *pk, A.POOL_MAX))
    ldc = _ldc(k, out_dtype)
    d = _stem_desc(A, A.MATH_I8, out_dtype, case, ldc, relu, float(np.float32(1) / s), monotone=monotone)
    got = _run_stem(A, d, x, wq, bias, scale, _torch_dt(out_dtype))
    assert (got[..., k:] == 0).all()
    np.testing.assert_array_equal(got[..., :k], want)


# 8-bit images normalised by mean 127.5 and a power-of-two scale, quantised by its inverse: every value u - 127.5 is
# a half step, from -127.5 to 127.5
IMG_MEAN, IMG_SCALE = [127.5] * 3, [2.0 ** -7] * 3


def tie_image(n, h, w):
    u8 = (np.arange(n * h * w * 3).reshape(n, h, w, 3) * 7 % 256).astype(np.uint8)
    assert len(np.unique(u8)) == 256
    return u8


@pytest.mark.parametrize("out", ["s8", "u8"])
def test_image_to_nhwc_quantisation_ties(out, oracle):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    from test_image_input_gpu import normalise
    n, h, w, c = 2, 19, 23, 3
    u8 = tie_image(n, h, w)
    x = normalise(u8, IMG_MEAN, IMG_SCALE, [0, 1, 2])
    s = np.float32(IMG_SCALE[0])
    unsigned = out == "u8"
    if not unsigned:
        assert_ties(x.astype(np.float64) / s, -128, 127, what="the normalised image")
    xt = np.ascontiguousarray(x.transpose(0, 2, 3, 1))
    want = oracle.quant_fp32_u8(xt, s) if unsigned else oracle.quant_fp32_s8(xt, s)
    inv = np.float32(1) / (s * (np.float32(127) / np.float32(255))) if unsigned else np.float32(1) / s
    fmt = A.image_desc(IMG_MEAN, IMG_SCALE)
    got = _dev_out((n, h, w, 16), _DT[out], 5)
    ud = dev(u8)
    A.check(A.load().b200_image_to_nhwc(C.byref(fmt), ptr(ud), ptr(got), _DT[out], n, c, h, w, 16, float(inv),
                                        stream_ptr()), "image")
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    np.testing.assert_array_equal(got[..., :c], want)
    assert (got[..., c:] == 0).all()


@pytest.mark.parametrize("out", ["f32", "s8"])
@pytest.mark.parametrize("pool", [(3, 2, 0), None], ids=["pool", "nopool"])
def test_stem_conv_image_quantisation_ties(pool, out, oracle):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    from test_image_input_gpu import _stem_desc, normalise
    n, h, w, c, k = 2, 40, 44, 3, 64
    case = (n, c, h, w, k, 7, 7, 2, 3, pool)
    u8 = tie_image(n, h, w)
    x = normalise(u8, IMG_MEAN, IMG_SCALE, [0, 1, 2])
    s = np.float32(IMG_SCALE[0])
    assert_ties(x.astype(np.float64) / s, -128, 127, what="the normalised image")
    wq = np.random.default_rng(19).integers(-127, 128, (k, c, 7, 7)).astype(np.int8)
    out_dtype = _DT[out]
    bias = np.zeros(k, np.float32)
    scale = np.ones(k, np.float32) if out_dtype == A.FLOAT else np.full(k, 1 / 1500.0, np.float32)
    xq = oracle.quant_fp32_s8(np.ascontiguousarray(x.transpose(0, 2, 3, 1)), s)
    want = oracle.conv_s8_nhwc_x86(xq, wq, bias, scale, out_dtype=out_dtype, stride=(2, 2), pad=(3, 3), relu=True)
    if pool is not None:
        pk = ((pool[0],) * 2, (pool[2],) * 2, (pool[1],) * 2)
        want = (oracle.pool_f32(want, *pk, A.POOL_MAX, nhwc=True) if out_dtype == A.FLOAT
                else oracle.pool_s8_nhwc(want, *pk, A.POOL_MAX))
    lib = A.load()
    ldc = _ldc(k, out_dtype)
    d = _stem_desc(A, A.MATH_I8, out_dtype, case, ldc, float(np.float32(1) / s))
    packed = np.zeros(lib.b200_stem_packed_weight_bytes(C.byref(d)), np.uint8)
    A.check(lib.b200_stem_pack_weights(C.byref(d), wq.ctypes.data_as(C.c_void_p), packed.ctypes.data_as(C.c_void_p)))
    got = _dev_out((n,) + want.shape[1:3] + (ldc,), out_dtype)
    fmt = A.image_desc(IMG_MEAN, IMG_SCALE)
    ud, wd, bd, sd = dev(u8), dev(packed), dev(bias), dev(scale)     # alive until the kernel has run
    A.check(lib.b200_stem_conv_run_image(C.byref(d), C.byref(fmt), ptr(ud), ptr(wd), ptr(bd), ptr(sd), ptr(got),
                                         stream_ptr()), "stem image")
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.cpu().numpy()[..., :k], want)


# ================================================================================ d. full-range pooling
# 256 channels. Channel j holds the value a_j on half of the pixels and a_j + 1 on the other half, as a checkerboard,
# so that every window with an even tap count averages to exactly a_j + 0.5; a_j covers the whole code range.
# Channels 254 and 255 are saturated planes: all -128 and all 127 for s8, all 0xFF for u8.
def pool_planes(n, h, w, unsigned):
    lo, hi = (0, 255) if unsigned else (-128, 127)
    a = lo + np.arange(256)
    chk = (np.add.outer(np.arange(h), np.arange(w)) % 2)[None, :, :, None]
    x = np.broadcast_to(a + chk, (n, h, w, 256)).astype(np.int16).copy()
    x[..., 254] = hi if unsigned else lo
    x[..., 255] = hi
    return x.astype(np.uint8 if unsigned else np.int8)


# (window h, window w, input h, input w): 255, 256, 257, 258 and 272 taps; non-global inputs leave ragged windows
POOL_WINDOWS = [(1, 255, 2, 600), (16, 16, 40, 37), (1, 257, 3, 520), (2, 129, 5, 300), (16, 17, 33, 40)]


def _pool_sums(x, wh, ww, glob):
    """Window sums of the full windows (stride = window) of a pool_planes tensor."""
    v = x.astype(np.float64)
    if glob:
        return v.sum((1, 2))
    nh, nw = x.shape[1] // wh, x.shape[2] // ww
    return v[:, :nh * wh, :nw * ww].reshape(x.shape[0], nh, wh, nw, ww, -1).sum((2, 4))


@pytest.mark.parametrize("ptype", [A.POOL_MAX, A.POOL_AVG_INC, A.POOL_AVG_EXC], ids=["max", "avg_inc", "avg_exc"])
@pytest.mark.parametrize("glob", [True, False], ids=["global", "strided"])
@pytest.mark.parametrize("window", POOL_WINDOWS, ids=lambda t: "%dx%d" % t[:2])
@pytest.mark.parametrize("unsigned", [True, False], ids=["u8", "s8"])
def test_pool_full_range(unsigned, window, glob, ptype, oracle):
    from test_pointwise_gpu import _pool
    wh, ww, h, w = window
    if glob:
        h, w = wh, ww
    n = 2
    x = pool_planes(n, h, w, unsigned)
    taps = wh * ww
    sums = _pool_sums(x, wh, ww, glob)
    peak = 255 * taps if unsigned else 128 * taps
    assert np.abs(sums).max() == peak, "a saturated plane must fill a whole window"
    if taps % 2 == 0 and ptype != A.POOL_MAX:
        assert_ties(sums / taps, *_BOUNDS[A.UINT8 if unsigned else A.INT8], what="the window averages")
    want = oracle.pool_s8_nhwc(x, (wh, ww), (0, 0), (wh, ww), ptype, global_pooling=glob)
    got = _pool(A.UINT8 if unsigned else A.INT8, (n, h, w, 256, (wh, ww), 0, (wh, ww), glob), ptype, x)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("pool_max", [0, 1], ids=["avg", "max"])
@pytest.mark.parametrize("unsigned", [True, False], ids=["u8", "s8"])
def test_head_pool_full_range(unsigned, pool_max, oracle):
    """The head's packed 16-bit average at its 256-pixel limit, on saturated and half-tie planes; 257 pixels of
    average pooling are refused."""
    m, c, n = 4, 256, 40
    x = pool_planes(m, 16, 16, unsigned)
    rng = np.random.default_rng(23)
    w = rng.integers(-127, 128, (n, c)).astype(np.int8)
    bias = rng.uniform(-2000, 2000, n).astype(np.float32)
    scale = np.full(n, 1.0 / 4000, np.float32)
    want_pool = oracle.pool_s8_nhwc(x, (16, 16), (0, 0), (16, 16), 2 - pool_max, global_pooling=True).reshape(m, c)
    if not pool_max:
        assert_ties(_pool_sums(x, 16, 16, True) / 256, *_BOUNDS[A.UINT8 if unsigned else A.INT8], at_least=4,
                    what="the head's averages")
    want = oracle.conv_s8_nhwc_x86(want_pool.reshape(m, 1, 1, c), w.reshape(n, c, 1, 1), bias, scale,
                                   out_dtype=A.FLOAT).reshape(m, n)
    pooled, logits = run_head(x, w, bias, scale, pool_max)
    np.testing.assert_array_equal(pooled, want_pool)
    np.testing.assert_array_equal(logits, want)
    x257 = pool_planes(m, 1, 257, unsigned)
    if pool_max:
        pooled, _ = run_head(x257, w, bias, scale, 1)
        np.testing.assert_array_equal(pooled, oracle.pool_s8_nhwc(x257, (1, 257), (0, 0), (1, 257), 1,
                                                                  global_pooling=True).reshape(m, c))
    else:
        run_head(x257, w, bias, scale, 0, expect=A.UNIMPL_ERROR)


# ================================================================================ e. eltwise, exhaustively
ELT_SCALES = [(0.5, 0.5), (0.25, 0.75), (0.1, 0.7), (1.0, 1.0), (2.0, -1.5)]


def _elt_pre(a, b, sa, sb):
    """The oracle's pre-rounding sum: two fp32 products, one fp32 add."""
    return np.float32(a.astype(np.float32) * np.float32(sa)) + np.float32(b.astype(np.float32) * np.float32(sb))


@functools.lru_cache(maxsize=None)
def eltwise_case(ua, ub, uo, relu, scales):
    """All 65536 (a, b) pairs, then a 15-element tail of ties and saturating pairs for the kernel's scalar loop."""
    from oracle import pyoracle as oracle
    sa, sb = scales
    ia, ib = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    a = ia.ravel().astype(np.uint8).view(np.uint8 if ua else np.int8)
    b = ib.ravel().astype(np.uint8).view(np.uint8 if ub else np.int8)
    out = A.UINT8 if uo else A.INT8
    lo, hi = _out_range(out, relu)
    pre = _elt_pre(a, b, sa, sb)
    if scales[0] in (0.5, 0.25):
        assert_ties(pre, lo, hi, what="eltwise %s" % (scales,))
    elif scales == (0.1, 0.7):
        # fma(b, sb, a * sa): the fp32 product a * sa plus the exact b * sb, rounded once
        fused = (np.float32(a.astype(np.float32) * np.float32(sa)).astype(np.float64) +
                 b.astype(np.float64) * np.float64(np.float32(sb))).astype(np.float32)
        sep = (roundf(fused) != roundf(pre)) & (pre > lo - 0.5) & (pre < hi + 0.5)
        assert sep.any(), "no pair separates fused from unfused arithmetic"
    else:
        # past every bound the input ranges can reach
        corners = [p * sa + q * sb for p in ((0, 255) if ua else (-128, 127)) for q in ((0, 255) if ub else (-128, 127))]
        assert max(corners) > hi + 0.5 or min(corners) < lo - 0.5, "eltwise %s cannot saturate" % (scales,)
        if max(corners) > hi + 0.5:
            assert (pre > hi + 0.5).any(), "eltwise %s must saturate above" % (scales,)
        if min(corners) < lo - 0.5:
            assert (pre < lo - 0.5).any(), "eltwise %s must saturate below" % (scales,)
    # the tail: ties (both signs and parities where there are any), then the extremes
    frac = np.abs(pre - np.trunc(pre)) == 0.5
    pick = []
    for cls in [(-1, 0), (-1, 1), (1, 0), (1, 1)]:
        idx = np.flatnonzero(frac & (np.sign(pre) == cls[0]) & (np.trunc(np.abs(pre)) % 2 == cls[1]) &
                             (pre > lo - 0.5) & (pre < hi + 0.5))
        pick += list(idx[:3])
    pick += [int(np.argmin(pre)), int(np.argmax(pre))]
    pick = (pick + list(range(15)))[:15]
    a = np.concatenate([a, a[pick]])
    b = np.concatenate([b, b[pick]])
    want = oracle.eltwise_sum_q8(a, b, sa, sb, out, relu=relu)
    return a, b, want


@pytest.mark.parametrize("scales", ELT_SCALES, ids=lambda s: "%g,%g" % s)
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("ua,ub,uo", [(False, False, False), (True, False, False), (True, True, True), (False, False, True),
                                      (True, False, True), (True, True, False)],
                         ids=["s8s8-s8", "u8s8-s8", "u8u8-u8", "s8s8-u8", "u8s8-u8", "u8u8-s8"])
def test_eltwise_all_pairs(ua, ub, uo, relu, scales):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    a, b, want = eltwise_case(ua, ub, uo, relu, scales)
    dt = lambda u: A.UINT8 if u else A.INT8
    ad, bd = dev(a), dev(b)
    for count in (65536, a.size):       # the 16-wide vector loop alone, then with the scalar tail
        out = _dev_out((count,), dt(uo), 7)
        A.check(A.load().b200_eltwise_run(dt(ua), dt(ub), dt(uo), A.ELT_SUM, ptr(ad), ptr(bd), ptr(out), count,
                                          float(scales[0]), float(scales[1]), int(relu), stream_ptr()))
        torch.cuda.synchronize()
        np.testing.assert_array_equal(out.cpu().numpy(), want[:count], err_msg="count %d" % count)


# ================================================================================ f. depthwise and fc epilogues
def dw_design(n, h, w, c, r, unsigned):
    """One nonzero tap (the centre one) per channel, of weight 1, 127 or -127; the channels take (bias, scale) pairs
    of the conv grid; every channel sees every input code."""
    lo = 0 if unsigned else -128
    p = np.arange(n * h * w).reshape(n, h, w, 1)
    x = ((p + 37 * np.arange(c)) % 256 + lo).astype(np.int16).astype(np.uint8 if unsigned else np.int8)
    tap = np.array([1, 127, -127, 1])[np.arange(c) % 4]
    wq = np.zeros((c, 1, r, r), np.int8)
    wq[:, 0, r // 2, r // 2] = tap
    gb, gs = grid_pairs()
    idx = (np.arange(c) * 7) % len(gb)
    return x, wq, gb[idx], gs[idx]


DW_KERNELS = {"row-3x3": (2, 29, 31, 96, 3, 1, 1), "row-3x3s2": (2, 29, 31, 96, 3, 2, 1),
              "vec-5x5": (2, 29, 31, 96, 5, 1, 1), "vec-3x3d2": (2, 29, 31, 96, 3, 1, 2),
              "tile-8": (2, 30, 37, 128, 3, 1, 1), "tile-4": (1, 29, 70, 64, 3, 1, 1)}   # (n, h, w, c, r, stride, dil)
DW_VARIANTS = {"s8_s8": (False, A.INT8, False), "u8_relu_u8": (True, A.UINT8, True), "u8_s8": (True, A.INT8, False),
               "s8_u8": (False, A.UINT8, False)}


@pytest.mark.parametrize("variant", list(DW_VARIANTS))
@pytest.mark.parametrize("kernel", list(DW_KERNELS))
def test_dwconv_epilogue_grid(kernel, variant, oracle):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    n, h, w, c, r, stride, dil = DW_KERNELS[kernel]
    unsigned, out_dtype, relu = DW_VARIANTS[variant]
    pad = (r - 1) * dil // 2
    x, wq, bias, scale = dw_design(n, h, w, c, r, unsigned)
    kw = dict(stride=(stride, stride), dil=(dil, dil), pad=(pad, pad), group=c)
    want = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, out_dtype=out_dtype, relu=relu, **kw)
    pre = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, out_dtype=A.FLOAT, **kw)
    lo, hi = _out_range(out_dtype, relu)
    assert_ties(pre, lo, hi, at_least=10, what=kernel)
    assert_clamps(pre, lo, hi, kernel)
    d = A.ConvDesc()
    d.math, d.in_dtype, d.out_dtype, d.res_dtype = A.MATH_I8, (A.UINT8 if unsigned else A.INT8), out_dtype, -1
    d.n, d.h, d.w, d.c, d.k, d.ldc, d.r, d.s = n, h, w, c, c, c, r, r
    d.pad_h = d.pad_w = pad
    d.stride_h = d.stride_w = stride
    d.dil_h = d.dil_w = dil
    d.relu = int(relu)
    wrsc = np.ascontiguousarray(np.transpose(wq[:, 0], (1, 2, 0)))
    out = _dev_out(want.shape, out_dtype)
    xd, wd, bd, sd = dev(x), dev(wrsc), dev(bias), dev(scale)     # alive until the kernel has run
    A.check(A.load().b200_dwconv_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), ptr(sd), ptr(out),
                                     stream_ptr()))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), want)


def fc_grid(unsigned):
    """16 rows whose accumulators x0 + 127 * x1 span the whole range, k = 32; every scale of the conv grid against
    biases in half steps over [-400, 400]."""
    lo, hi = (0, 255) if unsigned else (-128, 127)
    x0 = np.array([lo, hi, 0, 1, 3, 100, lo + 1, hi - 1, 50, 77, 2, 255 if unsigned else -1, 9, 120, 64, 33])
    x1 = np.array([lo, hi, 0, 0, 1, 2, 0, 1, hi, lo, 3, 0, 5, 0, 1, 0])
    x = np.zeros((16, 32), np.int16)
    x[:, 0], x[:, 1] = np.clip(x0, lo, hi), np.clip(x1, lo, hi)
    gs = np.unique(grid_pairs()[1])
    b = np.arange(-400, 400.5, 0.5, dtype=np.float32)
    bias = np.tile(b, len(gs)).astype(np.float32)
    scale = np.repeat(gs, len(b)).astype(np.float32)
    w = np.zeros((bias.size, 32), np.int8)
    w[:, 0], w[:, 1] = 1, 127
    return x.astype(np.uint8 if unsigned else np.int8), w, bias, scale


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("out", ["s8", "u8", "f32"])
@pytest.mark.parametrize("unsigned", [True, False], ids=["u8in", "s8in"])
def test_fc_stream_epilogue_grid(unsigned, out, relu, oracle):
    x, w, bias, scale = fc_grid(unsigned)
    m, k = x.shape
    n = w.shape[0]
    out_dtype = _DT[out]
    want = oracle.conv_s8_nhwc_x86(x.reshape(m, 1, 1, k), w.reshape(n, k, 1, 1), bias, scale, out_dtype=out_dtype,
                                   relu=relu).reshape(m, n)
    pre = oracle.conv_s8_nhwc_x86(x.reshape(m, 1, 1, k), w.reshape(n, k, 1, 1), bias, scale, out_dtype=A.FLOAT)
    if out_dtype != A.FLOAT:
        lo, hi = _out_range(out_dtype, relu)
        assert_ties(pre, lo, hi, what="fc grid")
        assert_clamps(pre, lo, hi, "fc grid")
    np.testing.assert_array_equal(run_fc(x, w, bias, scale, out_dtype, relu), want)
