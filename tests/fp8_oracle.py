"""The E4M3 (OCP e4m3fn) conv kind restated in numpy: codec, exact accumulation, epilogue and fused MAX pooling, as
include/b200_saber.h specifies them.

- Codec: a table of the 256 codes. Encoding rounds to nearest even on the finite grid and saturates to +-448 (the
  device's cvt.rn.satfinite.e4m3x2.f32); decoding is exact.
- Accumulation: every product of two E4M3 values is a multiple of 2^-18 below 448^2 < 2^17.7, so a float64 sum of up
  to 2^35 products is an integer below 2^53 in units of 2^-18: exact. The oracle's accumulator is that exact sum, and
  `conv` asserts the 2^53 bound.
- Epilogue: (acc + bias) * scale, fmaf(dec(res), sum_scale, .), relu to +0, enc -- each step an fp32 rounding.

No torch here: the generators run on machines without a GPU (tests/test_cpu_fp8.py checks the codec against
torch.float8_e4m3fn where torch is installed).
"""
import numpy as np

import float_exact as F
from se_oracle import fmaf

F32 = np.float32
MAX = 448.0
UNIT_LOG2 = -18                       # products of two codes are multiples of 2^-18


def _decode_table():
    t = np.zeros(256, np.float64)
    for c in range(256):
        s, e, m = c >> 7, (c >> 3) & 15, c & 7
        if e == 15 and m == 7:
            v = np.nan
        elif e == 0:
            v = m * 2.0 ** -9
        else:
            v = (1 + m / 8.0) * 2.0 ** (e - 7)
        t[c] = -v if s else v
    return t


DECODE = _decode_table()
_POS = DECODE[:127]                   # codes 0x00..0x7e: the non-negative finite values, increasing


def decode(codes):
    return DECODE[np.asarray(codes, np.uint8)]


def encode(x):
    """fp32 values -> uint8 codes: round to nearest even, saturate to +-448, NaN to 0x7f; -0.0 and negative values
    that round to zero keep the sign bit."""
    x = np.asarray(x, F32)
    a = np.abs(x.astype(np.float64))
    nan = np.isnan(a)
    a = np.minimum(np.where(nan, 0.0, a), MAX)
    hi = np.clip(np.searchsorted(_POS, a, side="left"), 0, 126)     # first grid value >= a
    lo = np.maximum(hi - 1, 0)
    d_lo, d_hi = a - _POS[lo], _POS[hi] - a
    code = np.where(d_lo < d_hi, lo, np.where(d_hi < d_lo, hi, np.where(lo % 2 == 0, lo, hi)))
    code = np.where(_POS[hi] == a, hi, code).astype(np.uint8)
    code = code | np.where(np.signbit(x), 0x80, 0).astype(np.uint8)
    return np.where(nan, np.uint8(0x7F), code).astype(np.uint8)


def conv(x_codes, w_codes, stride=(1, 1), pad=(0, 0), dil=(1, 1)):
    """NHWC codes [n][h][w][c] (*) KCRS codes: the exact float64 sum of the decoded products, asserting that the sum of
    their magnitudes stays below 2^53 units of 2^-18."""
    x, w = decode(x_codes), decode(w_codes)
    units = F.conv_f64(np.abs(x), np.abs(w), stride, pad, dil) * 2.0 ** -UNIT_LOG2
    assert units.size == 0 or units.max() < 2.0 ** 53, "the float64 sums are not exact (%g units)" % units.max()
    return F.conv_f64(x, w, stride, pad, dil)


def epilogue(acc, bias, scale, res_codes=None, sum_scale=1.0, relu=False, out_fp32=False):
    """acc [..., k] exact sums (fp32 on the device: the designed data keep them exact), bias / scale [k] fp32: the
    output codes (or fp32 values)."""
    a = np.asarray(acc, np.float64)
    assert (a.astype(F32).astype(np.float64) == a).all(), "the accumulator is not an fp32 number"
    f = (a.astype(F32) + np.asarray(bias, F32)).astype(F32)
    f = (f * np.asarray(scale, F32)).astype(F32)
    if res_codes is not None:
        f = fmaf(decode(res_codes).astype(F32), F32(sum_scale), f)
    if relu:
        f = np.where(f > 0, f, F32(0)).astype(F32)
    return f if out_fp32 else encode(f)


def max_pool(values, window, stride, pad, out_hw, codes=True):
    """MAX pooling of NHWC e4m3 codes (or fp32 values) as the fused pooling computes it: windows clipped to the input,
    visited row by row; the running element is replaced when its value (decoded, for codes) is below the next one's
    (r >= x ? r : x)."""
    key = decode if codes else (lambda v: v)
    n, h, w, c = values.shape
    ho, wo = out_hw
    out = np.zeros((n, ho, wo, c), values.dtype)
    for i in range(ho):
        for j in range(wo):
            hs, he = max(i * stride - pad, 0), min(i * stride - pad + window, h)
            ws, we = max(j * stride - pad, 0), min(j * stride - pad + window, w)
            acc = values[:, hs, ws].copy()
            first = True
            for y in range(hs, he):
                for xx in range(ws, we):
                    if first:
                        first = False
                        continue
                    v = values[:, y, xx]
                    acc = np.where(key(acc) >= key(v), acc, v)
            out[:, i, j] = acc
    return out


# ------------------------------------------------------------------------------------------------ designed data
# Codes of small integers times a power of two (x = X * 2^-4, w = W * 2^-3, |X|, |W| <= 8 are all E4M3 numbers), with
# the sum of |products| of every output at most 2^EXACT_BITS quanta (2^-7): every partial sum, in any order, is then a
# multiple of the quantum below 2^EXACT_BITS quanta, exact in an accumulator that keeps EXACT_BITS + 1 significant bits.
# test_fp8_gpu.py's probe measures how many the tensor cores keep and must find at least that.
EXACT_BITS = 12
X_EXP, W_EXP = -4, -3


def _sparse_ints(rng, shape, m, density):
    v = rng.integers(-m, m + 1, shape)
    return np.where(rng.random(shape) < density, v, 0)


def designed_case(geom, out_fp32, with_res, relu, key):
    """(x codes NHWC, w codes KCRS, bias, scale, res codes or None, sum_scale, expected output codes / fp32) for
    geom = (n, h, w, c, k, r, s, stride, pad_h, pad_w, dil). Channels of the epilogue table: j % 4 == 0 bias 0 and a
    power-of-two scale (many exact E4M3 ties), 1 a scale that saturates most values, 2 and 3 fp32 bias and scale with
    full mantissas."""
    n, h, w, c, k, r, s, stride, ph, pw, dil = geom
    rng = np.random.default_rng(F.seed("fp8", geom, out_fp32, with_res, relu, key))
    kw = dict(stride=(stride, stride), pad=(ph, pw), dil=(dil, dil))
    m = 8
    density = min(1.0, 2.0 ** EXACT_BITS / (c * r * s * 24.0))
    for _ in range(40):
        X = _sparse_ints(rng, (n, h, w, c), m, density)
        W = _sparse_ints(rng, (k, c, r, s), m, 1.0)
        worst = F.conv_f64(np.abs(X).astype(np.float64), np.abs(W).astype(np.float64), **kw).max()
        if worst <= 2 ** EXACT_BITS:
            break
        density *= 0.7
    else:
        raise AssertionError("no designed data within the bound for %s" % (geom,))
    x = encode((X * 2.0 ** X_EXP).astype(F32))
    wc = encode((W * 2.0 ** W_EXP).astype(F32))
    assert (decode(x) == X * 2.0 ** X_EXP).all() and (decode(wc) == W * 2.0 ** W_EXP).all()
    acc = conv(x, wc, **kw)
    units = F.conv_f64(np.abs(decode(x)), np.abs(decode(wc)), **kw) / 2.0 ** (X_EXP + W_EXP)
    assert units.max() <= 2 ** EXACT_BITS, units.max()
    assert (acc != 0).mean() > 0.3, "designed data too sparse"
    j = np.arange(k)
    u = 2.0 ** -(X_EXP + W_EXP)                       # one quantum of acc -> 1.0
    bias = np.where(j % 4 == 0, 0.0, rng.uniform(-32, 32, k) * 2.0 ** (X_EXP + W_EXP)).astype(F32)
    scale = np.where(j % 4 == 0, u * 2.0 ** -(j % 7), np.where(j % 4 == 1, u * 64.0, rng.uniform(0.01, 0.5, k) * u))
    scale = scale.astype(F32)
    res, sum_scale = None, 1.0
    if with_res:
        oh = (h + 2 * ph - dil * (r - 1) - 1) // stride + 1
        ow = (w + 2 * pw - dil * (s - 1) - 1) // stride + 1
        res = encode(rng.uniform(-300, 300, (n, oh, ow, k)).astype(F32))
        sum_scale = float(F32(0.37))
    want = epilogue(acc, bias, scale, res, sum_scale, relu, out_fp32)
    return x, wc, bias, scale, res, sum_scale, want
