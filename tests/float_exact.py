"""Designed data with exact sums for the float kernels, and the expected outputs from the CPU oracle.

Inputs are integers times a power of two. When, for every output, the sum of |x * w| over its taps plus |residual| is
at most 2^22 times the quantum of the products, every partial sum is an exact fp32 number in any summation order: the
im2col and slab k loops, split-K partial sums, and the tensor core's aligned accumulation. The only roundings left are
`+ bias`, `* neg_slope` and the store, so a correct kernel gives the oracle's bits exactly, and for f16 outputs the bits
of numpy's round-half-to-even conversion of them. Every generator checks that bound (assert_exact) and asserts its
own coverage, so an edit that breaks the bound or makes a case vacuous fails on the CPU as well
(tests/test_cpu_float_exact.py).

No torch here: the generators run on machines without a GPU.
"""
import functools
import warnings
import zlib

import numpy as np

from anakin_b200 import saber_abi as A

EXACT_BITS = 22                      # 2 bits of margin below fp32's 24
TF32_MASK = np.uint32(0xFFFFE000)    # sign, exponent and the top 10 mantissa bits


def oracle():
    from oracle import pyoracle
    return pyoracle


def seed(*key):
    """A seed that is the same on every run (hash() of strings changes with PYTHONHASHSEED), so that a mismatch on
    the GPU can be reproduced from the same data."""
    return zlib.crc32(repr(key).encode())


# ------------------------------------------------------------------------------------------------ exactness bound
def _tap_slices(n, h, w, r, s, stride, pad, dil):
    oh = (h + 2 * pad[0] - dil[0] * (r - 1) - 1) // stride[0] + 1
    ow = (w + 2 * pad[1] - dil[1] * (s - 1) - 1) // stride[1] + 1
    for ky in range(r):
        for kx in range(s):
            y0, x0 = ky * dil[0], kx * dil[1]
            yield ky, kx, (slice(None), slice(y0, y0 + (oh - 1) * stride[0] + 1, stride[0]),
                           slice(x0, x0 + (ow - 1) * stride[1] + 1, stride[1]))


def conv_f64(x, w, stride=(1, 1), pad=(0, 0), dil=(1, 1)):
    """NHWC x [n][h][w][c] (*) KCRS w in float64. Exact for the dyadic operands used here as long as every sum stays
    below 2^53 times its quantum, which assert_exact's 2^22 bound implies."""
    n, h, wd, c = x.shape
    k, _, r, s = w.shape
    xp = np.zeros((n, h + 2 * pad[0], wd + 2 * pad[1], c), np.float64)
    xp[:, pad[0]:pad[0] + h, pad[1]:pad[1] + wd] = x
    acc = None
    for ky, kx, sl in _tap_slices(n, h, wd, r, s, stride, pad, dil):
        t = xp[sl] @ np.asarray(w[:, :, ky, kx], np.float64).T
        acc = t if acc is None else acc + t
    return acc


def assert_exact(abs_sum, quantum, what=""):
    """abs_sum: per-output sum of |x * w| (+ |residual|), all multiples of `quantum`; asserts the 2^22 bound."""
    units = np.asarray(abs_sum, np.float64) / quantum
    assert (units == np.rint(units)).all(), "%s: an operand is not a multiple of the quantum" % what
    assert units.max() <= 2.0 ** EXACT_BITS, "%s: the sums are not exact in fp32 (%d > 2^%d quanta)" % (
        what, units.max(), EXACT_BITS)
    return units.max()


def quantum_of(*arrays):
    """The largest power of two that divides every nonzero element of every array (all must be dyadic)."""
    e = None
    for a in arrays:
        v = np.abs(np.asarray(a, np.float64).ravel())
        v = v[v != 0]
        if v.size:
            m, ex = np.frexp(v)                        # v = m * 2^ex, m in [0.5, 1)
            mi = (m * 2.0 ** 53).astype(np.int64)      # exact: the integer mantissa
            low = np.log2((mi & -mi).astype(np.float64)).astype(np.int64)      # its lowest set bit
            lo = int((ex - 53 + low).min())
            e = lo if e is None else min(e, lo)
    return 1.0 if e is None else 2.0 ** e


def conv_quantum(x, w, res=None):
    """Per output channel: the quantum of its products (and of its residual)."""
    qx = quantum_of(x)
    q = np.array([qx * quantum_of(w[j]) for j in range(w.shape[0])])
    if res is not None:
        q = np.minimum(q, [quantum_of(res[..., j]) for j in range(w.shape[0])])
    return q


def check_conv_exact(x, w, res=None, stride=(1, 1), pad=(0, 0), dil=(1, 1), what="", quantum=None):
    """Asserts the exactness bound of a conv on these operands; returns the largest sum in quanta. `quantum` overrides
    the per-channel product of the operands' quanta (which is too fine where operands come in hi / lo planes)."""
    s = conv_f64(np.abs(np.asarray(x, np.float64)), np.abs(np.asarray(w, np.float64)), stride, pad, dil)
    if res is not None:
        s = s + np.abs(np.asarray(res, np.float64))
    return assert_exact(s, conv_quantum(x, w, res) if quantum is None else quantum, what)


# ------------------------------------------------------------------------------------------------ rounding classes
def f16_ties(v):
    """(is a tie, rounds up in magnitude) of fp32 values against the f16 grid, subnormals included."""
    v = np.asarray(v, np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        h = v.astype(np.float16)
        d = v.astype(np.float64) - h.astype(np.float64)
        other = np.nextafter(h, np.where(d > 0, np.float16(np.inf), np.float16(-np.inf)).astype(np.float16))
        gap = np.abs(other.astype(np.float64) - h.astype(np.float64))
    tie = np.isfinite(h) & np.isfinite(other) & (d != 0) & (2 * np.abs(d) == gap)
    up = np.abs(h.astype(np.float64)) > np.abs(v.astype(np.float64))
    return tie, up


def assert_f16_classes(pre, at_least=20, what="", signs=(-1, 1), edges=True):
    """Exact f16 ties of the given signs and both rounding directions, values one fp32 ulp either side of ties, values
    past 65504 up to overflow, and subnormal ties, among the fp32 values `pre` before the f16 store."""
    pre = np.asarray(pre, np.float32).ravel()
    tie, up = f16_ties(pre)
    counts = {(sg, u): int((tie & (np.sign(pre) == sg) & (up == u)).sum()) for sg in signs for u in (False, True)}
    for key, n in counts.items():
        assert n >= at_least, "%s: too few f16 ties of sign %d, rounding %s: %s" % (what, key[0], "up" if key[1] else
                                                                                  "down", counts)
    for direction in (np.float32(np.inf), np.float32(-np.inf)):
        near = f16_ties(np.nextafter(pre, direction))[0] & ~tie
        assert near.sum() >= at_least, "%s: too few values one fp32 ulp beside an f16 tie" % what
    sub = tie & (np.abs(pre) < 2.0 ** -14)
    assert sub.sum() >= at_least, "%s: too few ties among f16 subnormals (%d)" % (what, sub.sum())
    a = np.abs(pre.astype(np.float64))
    assert ((a > 65504) & (a < 65520)).any(), "%s: nothing above 65504 that stays finite" % what
    assert (a >= 65520).any(), "%s: nothing that overflows to inf" % what
    if edges:      # the overflow threshold itself, and one fp32 ulp below it
        assert (a == 65520).any(), "%s: 65520 is missing" % what
        assert (a == np.float64(np.nextafter(np.float32(65520), np.float32(0)))).any(), "%s: no 65520 - 1 ulp" % what
    return counts


def f32_ties(exact):
    """Exact float64 values that lie halfway between two adjacent fp32 numbers."""
    e = np.asarray(exact, np.float64)
    f = e.astype(np.float32)
    d = e - f.astype(np.float64)
    other = np.nextafter(f, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    return (d != 0) & (2 * np.abs(d) == np.abs(other.astype(np.float64) - f.astype(np.float64)))


def f16_store(v):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.asarray(v, np.float32).astype(np.float16)


# ------------------------------------------------------------------------------------------------ dense exact data
# (n, h, w, c, k, r, stride, pad, dil); the shapes of test_conv_gpu.py's F_CASES, SPLIT_CASES and PERSISTENT_CASES
DENSE_F_CASES = [
    (1, 12, 12, 16, 32, 3, 1, 1, 1),
    (3, 21, 21, 8, 8, 3, 2, 1, 1),
    (2, 24, 24, 64, 64, 1, 1, 0, 1),
    (1, 36, 36, 32, 48, 3, 1, 2, 2),
    (2, 28, 28, 128, 128, 3, 1, 1, 1),
    (1, 56, 56, 64, 64, 1, 2, 0, 1),
    (1, 40, 40, 4, 64, 7, 2, 3, 1),
    (1, 14, 14, 256, 200, 3, 1, 1, 1),    # k ragged against every tile width
]

# name: (math kind, output, residual); the f16 kind alone stores and reads half
DENSE_VARIANTS = {
    "f16_h": ("f16", A.HALF, None),
    "f16_h_res-h": ("f16", A.HALF, A.HALF),
    "f16_h_res-f": ("f16", A.HALF, A.FLOAT),
    "f16_f": ("f16", A.FLOAT, None),
    "f16_f_res-h": ("f16", A.FLOAT, A.HALF),
    "f16_f_res-f": ("f16", A.FLOAT, A.FLOAT),
    "tf32x3_f": ("tf32x3", A.FLOAT, None),
    "tf32x3_f_res-f": ("tf32x3", A.FLOAT, A.FLOAT),
}

MATH = {"f16": A.MATH_F16, "tf32x3": A.MATH_TF32X3}
IN_DT = {"f16": A.HALF, "tf32x3": A.FLOAT}
DENSE_EX, DENSE_EW = -4, -3         # x = X * 2^-4, w = W * 2^-3: products are multiples of 2^-7
RES_MAX = 2048                      # |residual| <= 2048 quanta: exact in f16 at 2^-7


def es(dt):
    return 2 if dt == A.HALF else (1 if dt in (A.INT8, A.UINT8) else 4)


def ldc_for(k, out_dt, res_dt=None):
    """A row pitch above k (padding channels to keep untouched), 16-byte aligned for the output and the residual."""
    al = 16 // min(es(out_dt), es(res_dt) if res_dt is not None else 4)
    return (k + al - 1) // al * al + al


def in_channels(math, c, r):
    """(real channels, channels of the NHWC buffer): the f16 kind needs 8-channel rows, the stem-like 7x7 has 3 real."""
    c_real = 3 if r == 7 else c
    if math == "f16" and c % 8:
        c = 8
    return c_real, c


def full_geom(case):
    """(n, h, w, c, k, r, s, stride, pad_h, pad_w, dil) of a case in test_conv_gpu.py's F_CASES form
    (n, h, w, c, k, r, stride, pad, dil) or in this long form."""
    if len(case) == 9:
        n, h, w, c, k, r, stride, pad, dil = case
        return n, h, w, c, k, r, r, stride, pad, pad, dil
    return case


def dense_magnitude(kk):
    """The largest operand magnitude m (|X|, |W| <= m, m <= 15) with kk * m^2 + RES_MAX within the bound."""
    m = int(np.sqrt((2 ** EXACT_BITS - RES_MAX) / kk))
    return max(1, min(15, m))


@functools.lru_cache(maxsize=None)
def dense_case(case, variant, relu=True, neg_slope=0.1):
    """(x, w, bias, residual, expected) of one dense exact case. x and w are in the kind's operand type (f16 for the
    f16 kind), the residual in its dtype; `expected` is in the output dtype."""
    math, out_dt, res_dt = DENSE_VARIANTS[variant]
    n, h, w, c, k, r, s, stride, ph, pw, dil = full_geom(case)
    c_real, _ = in_channels(math, c, r)
    rng = np.random.default_rng(seed(case, variant))
    m = dense_magnitude(c_real * r * s)
    x = (rng.integers(-m, m + 1, (n, h, w, c_real)) * 2.0 ** DENSE_EX).astype(np.float32)
    wt = (rng.integers(-m, m + 1, (k, c_real, r, s)) * 2.0 ** DENSE_EW).astype(np.float32)
    bias = rng.uniform(-4, 4, k).astype(np.float32)       # full 24-bit mantissas: the + bias rounds
    oh = (h + 2 * ph - dil * (r - 1) - 1) // stride + 1
    ow = (w + 2 * pw - dil * (s - 1) - 1) // stride + 1
    res = None
    if res_dt is not None:
        res = (rng.integers(-RES_MAX, RES_MAX + 1, (n, oh, ow, k)) * 2.0 ** (DENSE_EX + DENSE_EW)).astype(np.float32)
    kw = dict(stride=(stride, stride), pad=(ph, pw), dil=(dil, dil))
    check_conv_exact(x, wt, res, what="dense %s %s" % (case, variant), **kw)
    want = oracle().conv_f32_nhwc(x, wt, bias, residual=res, beta=1.0, relu=relu, neg_slope=neg_slope, **kw)
    assert (want != np.rint(want)).mean() > 0.5 and (want < 0).any() and (want > 0).any()
    if out_dt == A.HALF:
        # the data must reach the f16 store's rounding: most values are not f16 numbers
        assert (f16_store(want).astype(np.float32) != want).mean() > 0.5
        want = f16_store(want)
    if math == "f16":
        x, wt = x.astype(np.float16), wt.astype(np.float16)
    if res_dt == A.HALF:
        r16 = res.astype(np.float16)
        assert (r16.astype(np.float32) == res).all(), "the residual must be exact in f16"
        res = r16
    return x, wt, bias, res, want


# ------------------------------------------------------------------------------------------------ float epilogue grid
# A 1x1 conv (or the centre tap of a padded 3x3) over 65536 pixels: channel 0 carries X0 * 2^-12, channel 1 carries
# X1 * 2^-4, for every pair (X0, X1) of [-128, 127]^2. Output channel j has both weights 2^(s_j + 12), so its
# accumulator is 2^s_j * (X0 + 256 X1): every multiple of 2^s_j in [-32896, 32639] * 2^s_j, exactly once. The
# channels form a table of (s_j, bias_j): unit exponents from f16-subnormal scales (2^-26: ties among subnormals) to
# 2^2 (past 65504 to inf), biases of 0, +-1 fp32 ulp of the channel's typical value, half a unit, and full 24-bit
# mantissas (where (acc + res) + bias and (acc + bias) + res round differently).
GRID_H, GRID_W, GRID_C, GRID_K = 128, 512, 16, 200     # 16 channels: 32-byte f16 rows, as the slab kernel needs
GRID_S = [-26, -23, -20, -16, -12, -9, -6, -3, 0, 2]


def grid_table():
    rows = []
    for s in GRID_S:
        u = 2.0 ** s
        rows += [(s, 0.0), (s, u * 2.0 ** -8), (s, -u * 2.0 ** -8), (s, u / 2),
                 (s, float(np.float32(1 / 3)) * u * 2.0 ** 13), (s, -float(np.float32(0.7)) * u * 2.0 ** 12)]
    rows += [(2, -2.0 ** -8), (2, 2.0 ** -8), (1, 0.0), (1, 2.0 ** -9)]
    s = np.array([r[0] for r in rows] * (GRID_K // len(rows) + 1))[:GRID_K]
    b = np.array([r[1] for r in rows] * (GRID_K // len(rows) + 1))[:GRID_K]
    b = np.where((np.arange(GRID_K) // len(rows)) % 2 == 1, -b, b)      # the second copy of the table negates biases
    assert (np.float64(np.float32(b)) == b).all()
    return s.astype(np.int64), b.astype(np.float32)


def grid_input():
    p = np.arange(GRID_H * GRID_W)
    x = np.zeros((1, GRID_H, GRID_W, GRID_C), np.float32)
    x[0, ..., 0] = ((p % 256 - 128) * 2.0 ** -12).reshape(GRID_H, GRID_W)
    x[0, ..., 1] = ((p // 256 - 128) * 2.0 ** -4).reshape(GRID_H, GRID_W)
    return x


def grid_weights(r):
    s, _ = grid_table()
    w = np.zeros((GRID_K, GRID_C, r, r), np.float32)
    w[:, 0, r // 2, r // 2] = 2.0 ** (s + 12)
    w[:, 1, r // 2, r // 2] = 2.0 ** (s + 12)
    return w


def grid_residual(dt):
    """Per pixel and channel 4 * R * 2^s_j, |R| <= 500: exact in f16 down to s_j = -26."""
    s, _ = grid_table()
    p = np.arange(GRID_H * GRID_W)[:, None]
    j = np.arange(GRID_K)[None, :]
    v = (4 * ((p * 5 + j * 3) % 1001 - 500) * 2.0 ** s[None, :]).astype(np.float32)
    v = v.reshape(1, GRID_H, GRID_W, GRID_K)
    return v.astype(np.float16) if dt == A.HALF else v


# name: (math kind, output, residual, relu, neg_slope)
GRID_VARIANTS = {
    "f16_h": ("f16", A.HALF, None, False, 0.0),
    "f16_h_relu0": ("f16", A.HALF, None, True, 0.0),
    "f16_h_res-h_leaky": ("f16", A.HALF, A.HALF, True, 0.1),
    "f16_h_res-f": ("f16", A.HALF, A.FLOAT, False, 0.0),
    "f16_f_res-f": ("f16", A.FLOAT, A.FLOAT, False, 0.0),
    "tf32x3_f_res-f_leaky": ("tf32x3", A.FLOAT, A.FLOAT, True, 0.1),
    "tf32x3_f_res-f_relu0": ("tf32x3", A.FLOAT, A.FLOAT, True, 0.0),
}


@functools.lru_cache(maxsize=None)
def grid_case(variant):
    """(x, bias, residual, expected) of one grid variant, after checking its coverage; the weights are grid_weights(r)
    (the 1x1 and the padded 3x3's centre tap have the same sums)."""
    math, out_dt, res_dt, relu, slope = GRID_VARIANTS[variant]
    x = grid_input()
    s, bias = grid_table()
    w = grid_weights(1)
    res = grid_residual(res_dt) if res_dt is not None else None
    res32 = res.astype(np.float32) if res is not None else None
    check_conv_exact(x, w, res32, what="grid " + variant)
    o = oracle()
    pre = o.conv_f32_nhwc(x, w, bias, residual=res32, relu=relu, neg_slope=slope)
    acc = conv_f64(x, w)
    assert np.array_equal(np.unique(acc[..., 0]), (np.arange(-32896, 32640) * 2.0 ** s[0])), "not every accumulator"
    if out_dt == A.HALF:
        assert_f16_classes(pre, what=variant, signs=(1,) if relu else (-1, 1), edges=res is None)
        want = f16_store(pre)
    else:
        exact = acc + (res32 if res32 is not None else 0) + bias.astype(np.float64)
        assert f32_ties(exact).sum() >= 100, "%s: too few fp32 ties at the + bias" % variant
        want = pre
    if relu and slope == 0.0:
        z = (want == 0) & np.signbit(want)
        assert z.sum() >= 1000, "%s: relu must give -0.0 for negative values" % variant
    if res is not None:
        # the epilogue's order: (acc + res) + bias, which rounds differently from (acc + bias) + res here
        a32 = acc.astype(np.float32)
        order = np.float32(a32 + res32) + bias
        other = np.float32(a32 + bias) + res32
        assert (order != other).sum() >= 1000, "%s: no value separates the two orders of the epilogue" % variant
    return x, bias, res, want


# ------------------------------------------------------------------------------------------------ 3xTF32 terms
# x = sign * (Xh * 2^e + Xl * 2^(e - 10)), Xh in [8, 15], Xl in [1, 7] (weights: Wl in [0, 7]): the tf32 split keeps the
# top 11 significant bits, so hi = sign * Xh * 2^e and lo = sign * Xl * 2^(e - 10), exactly. In units of
# u = 2^(ex + ew - 10) a tap's three products are Xh Wh 2^10, Xl Wh and Xh Wl (lo * lo = Xl Wl 2^-10 is left out): at
# most 230610 units, so 8 taps stay within 2^22 units and every sum of the three-term products is exact.
X3_EX, X3_EW, X3_TAPS = -3, -5, 8


def split_operand(rng, shape, e, lo_min):
    hi = rng.integers(8, 16, shape).astype(np.float64)
    lo = rng.integers(lo_min, 8, shape).astype(np.float64)
    sign = np.where(rng.integers(0, 2, shape) == 1, -1.0, 1.0)
    v = (sign * (hi * 2.0 ** e + lo * 2.0 ** (e - 10))).astype(np.float32)
    assert (v.astype(np.float64) == sign * (hi * 2.0 ** e + lo * 2.0 ** (e - 10))).all()
    return v


def tf32_hi(a):
    """numpy's restatement of the split: the same mask, sign-magnitude truncation."""
    return (np.ascontiguousarray(a, np.float32).view(np.uint32) & TF32_MASK).view(np.float32)


def tf32_lo(a):
    a = np.ascontiguousarray(a, np.float32)
    return (a - tf32_hi(a)).astype(np.float32)


def sparse_weights(rng, k, c, r, s, taps=X3_TAPS):
    """At most `taps` nonzero taps per output channel; channel j takes the reduction positions j + t * k (mod the
    reduction length), so that every position is hit by some channel when k * taps covers it."""
    kk = c * r * s
    flat = np.zeros((k, kk), np.float32)
    vals = split_operand(rng, (k, taps), X3_EW, 0)
    for t in range(taps):
        flat[np.arange(k), (np.arange(k) + t * k) % kk] = vals[:, t]
    # reduction index order (r, s, c) is the kernels' im2col order: position p = (ky * s + kx) * c + ci
    w = flat.reshape(k, r, s, c).transpose(0, 3, 1, 2)
    return np.ascontiguousarray(w)


def x3_expected_operands(x, w):
    """Operands whose plain conv is the three-term sum: [xh | xl | xh] (*) [wh | wh | wl] over 3c channels."""
    xs = np.concatenate([tf32_hi(x), tf32_lo(x), tf32_hi(x)], axis=-1)
    ws = np.concatenate([tf32_hi(w), tf32_hi(w), tf32_lo(w)], axis=1)
    return xs, ws


def x3_data(case):
    """(x, w, bias) of a split-term case: dense activations that all have low parts, sparse weights that mostly do.
    case = (n, h, w, c, k, r, s, stride, pad)."""
    n, h, wd, c, k, r, s, stride, pad = case
    rng = np.random.default_rng(seed(case, "x3"))
    x = split_operand(rng, (n, h, wd, c), X3_EX, 1)
    w = sparse_weights(rng, k, c, r, s)
    return x, w, rng.uniform(-1, 1, k).astype(np.float32)


# The share of outputs that must separate the kernels' result from each wrong one. On the designed data the two cross
# terms and the single pass each separate more than 0.99 of the outputs, and the full product about 0.8: lo * lo is a
# small term, which the rounding at + bias absorbs on the rest.
X3_SEPARATE = {"Alo*Whi": 0.9, "Ahi*Wlo": 0.9, "single pass": 0.9, "full product": 0.6}


def x3_outputs(x, w, bias, kw):
    """(the fp32 output of the three-term sum, {wrong result: its fp32 output}), from exact float64 sums of the four
    products: each sum is exact in fp32 too, so the + bias rounds once."""
    xh, xl, wh, wl = tf32_hi(x), tf32_lo(x), tf32_hi(w), tf32_lo(w)
    hh, lh, hl, ll = (conv_f64(a, b, **kw) for a, b in ((xh, wh), (xl, wh), (xh, wl), (xl, wl)))
    out = lambda s: (s + bias.astype(np.float64)).astype(np.float32)
    wrong = {"Alo*Whi": out(hh + hl), "Ahi*Wlo": out(hh + lh), "single pass": out(hh),
             "full product": out(hh + lh + hl + ll)}
    return out(hh + lh + hl), wrong


def x3_expected(x, w, bias, stride, pad, taps=X3_TAPS):
    """The expected fp32 output of a split-term case, Ahi Whi + Alo Whi + Ahi Wlo, after checking that the data shows
    every term. Data in which a term vanishes (no activation or no weight low parts) is refused. `taps`: the weights'
    nonzero taps per output channel at most (sparse_weights)."""
    k = w.shape[0]
    kw = dict(stride=(stride, stride), pad=(pad, pad))
    xs, ws = x3_expected_operands(x, w)
    # every product of the three planes is a multiple of 2^(ex + ew - 10)
    check_conv_exact(xs, ws, what="x3", quantum=2.0 ** (X3_EX + X3_EW - 10), **kw)
    three, wrong = x3_outputs(x, w, bias, kw)
    o = oracle()
    assert np.array_equal(three, o.conv_f32_nhwc(xs, ws, bias, **kw))
    # many fp32 outputs separate the three-term sum from the sum without each cross term, from the single tf32 pass
    # and from the full product (with lo * lo)
    for name, v in wrong.items():
        share = (v != three).mean()
        assert share > X3_SEPARATE[name], "only %.2f of the outputs separate the three-term sum from the %s" % (share, name)
    # every landed A tile is split, and every reduction position meets a weight
    assert (tf32_lo(x) != 0).all(), "every activation must have a low part"
    nz = (w != 0).reshape(k, -1)
    assert nz.sum(1).max() <= taps and nz.any(0).all(), "every reduction position must be hit by some channel"
    assert (tf32_lo(w)[w != 0] != 0).mean() > 0.75, "most weight taps must have a low part"
    return three


@functools.lru_cache(maxsize=None)
def x3_case(case):
    """(x, w, bias, expected fp32 output) of a split-term case. case = (n, h, w, c, k, r, s, stride, pad)."""
    x, w, bias = x3_data(case)
    return x, w, bias, x3_expected(x, w, bias, case[7], case[8])


# wgmma .tf32 truncates its fp32 operands to their top 11 significant bits, and 3xTF32 hands it lo = x - hi, which keeps
# up to 13. On activations x = sign * (H * 2^13 + L) * 2^q, H in [2^10, 2^11), L in [2^12, 2^13), the low part has 13
# significant bits and the tensor core multiplies L with its last two bits cleared. Weights are one power of two per
# output channel (no low part), so each output is (hi + trunc(lo)) * w + bias: below 2^22 quanta of 4 * 2^q * w. (A
# 12-bit low part would halve the quantum and need 2^23.)
TRUNC_CASE = (1, 8, 8, 64, 64)        # a 1x1 conv: n, h, w, c, k


def tf32_nearest(a):
    """a rounded to 11 significant bits, to nearest (ties away from zero) instead of truncated."""
    a = np.ascontiguousarray(a, np.float32)
    return ((a.view(np.uint32).astype(np.uint64) + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)


@functools.lru_cache(maxsize=None)
def x3_trunc_case():
    """(x, w, bias, expected fp32 output) of the truncated low plane, Ahi Whi + trunc(Alo) Whi + Ahi Wlo, after
    checking that rounding the low parts to nearest would change most outputs."""
    n, h, wd, c, k = TRUNC_CASE
    rng = np.random.default_rng(seed(TRUNC_CASE, "trunc"))
    hi = rng.integers(2 ** 10, 2 ** 11, (n, h, wd, c)).astype(np.float64)
    lo = rng.integers(2 ** 12, 2 ** 13, (n, h, wd, c))
    lo = np.where(rng.integers(0, 4, lo.shape) > 0, lo | 3, lo).astype(np.float64)   # mostly 0b11 cleared
    sign = np.where(rng.integers(0, 2, lo.shape) == 1, -1.0, 1.0)
    q = X3_EX - 23
    x = (sign * (hi * 2.0 ** 13 + lo) * 2.0 ** q).astype(np.float32)
    assert (x.astype(np.float64) == sign * (hi * 2.0 ** 13 + lo) * 2.0 ** q).all()
    assert (tf32_lo(x).astype(np.float64) == sign * lo * 2.0 ** q).all(), "the low parts must have 13 significant bits"
    w = np.zeros((k, c, 1, 1), np.float32)
    w[np.arange(k), np.arange(k) % c, 0, 0] = np.where(rng.integers(0, 2, k) == 1, -1.0, 1.0) * 2.0 ** X3_EW
    bias = (rng.uniform(-1, 1, k) * 2.0 ** (X3_EX + X3_EW - 2)).astype(np.float32)   # small: + bias keeps lo's bits
    xt = tf32_hi(x) + tf32_hi(tf32_lo(x))           # exact: 22 significant bits
    check_conv_exact(xt, w, what="x3 trunc", quantum=2.0 ** (q + 2 + X3_EW))
    o = oracle()
    want = o.conv_f32_nhwc(xt, w, bias)
    assert np.array_equal(want, (conv_f64(xt, w) + bias.astype(np.float64)).astype(np.float32))
    nearest = o.conv_f32_nhwc(tf32_hi(x) + tf32_nearest(tf32_lo(x)), w, bias)
    assert (nearest != want).mean() > 0.5, "truncating the low parts and rounding them to nearest must differ"
    return x, w, bias, want


# ------------------------------------------------------------------------------------------------ stem inputs
def f16_tie_inputs(shape, rng):
    """fp32 values on exact f16 half-ulp ties in [1, 2) and (-2, -1], both parities of the lower neighbour, plus
    values one fp32 ulp either side of ties; the f16 conversion rounds half to even."""
    k = rng.integers(0, 1024, shape)
    sign = np.where(rng.integers(0, 2, shape) == 1, -1.0, 1.0)
    v = (sign * (1.0 + (k + 0.5) * 2.0 ** -10)).astype(np.float32)
    sel = rng.integers(0, 8, shape)
    v = np.where(sel == 0, np.nextafter(v, np.float32(np.inf)), v)
    v = np.where(sel == 1, np.nextafter(v, np.float32(-np.inf)), v)
    return v.astype(np.float32)


def assert_tie_inputs(v, at_least=50):
    tie, up = f16_ties(v)
    for sg in (-1, 1):
        for u in (False, True):
            n = (tie & (np.sign(v) == sg) & (up == u)).sum()
            assert n >= at_least, "too few input ties of sign %d, rounding %s (%d)" % (sg, u, n)
    near = f16_ties(np.nextafter(v, np.float32(np.inf)))[0] | f16_ties(np.nextafter(v, np.float32(-np.inf)))[0]
    assert (near & ~tie).sum() >= at_least


@functools.lru_cache(maxsize=None)
def stem_case(case, math):
    """(x NCHW fp32, weight operand, bias, expected NHWC before any pooling) of the stem.
    case = (n, c, h, w, k, r, s, stride, pad, pool)."""
    n, c, h, wd, k, r, s, stride, pad, pool = case
    rng = np.random.default_rng(seed(case, math))
    kw = dict(stride=(stride, stride), pad=(pad, pad))
    bias = rng.uniform(-1, 1, k).astype(np.float32)
    o = oracle()
    if math == "f16":
        x = f16_tie_inputs((n, c, h, wd), rng)
        assert_tie_inputs(x)
        w = (rng.integers(-7, 8, (k, c, r, s)) * 2.0 ** -3).astype(np.float32)
        xs = np.ascontiguousarray(x.transpose(0, 2, 3, 1)).astype(np.float16).astype(np.float32)
        check_conv_exact(xs, w, what="stem f16", **kw)
        want = o.conv_f32_nhwc(xs, w, bias, relu=True, neg_slope=0.1, **kw)
        # rounding the inputs toward zero or away from it instead would change most outputs
        rz = np.trunc(np.ascontiguousarray(x.transpose(0, 2, 3, 1)).astype(np.float64) * 1024) / 1024
        assert (o.conv_f32_nhwc(rz.astype(np.float32), w, bias, relu=True, neg_slope=0.1, **kw) != want).mean() > 0.5
        return x, w.astype(np.float16), bias, f16_store(want)
    xn, w, b, want = x3_case((n, h, wd, c, k, r, s, stride, pad))
    want = o.conv_f32_nhwc(*x3_expected_operands(xn, w), b, relu=True, neg_slope=0.1, **kw)
    return np.ascontiguousarray(xn.transpose(0, 3, 1, 2)), w, b, want


# ------------------------------------------------------------------------------------------------ fc_stream
FC_N = 200


@functools.lru_cache(maxsize=None)
def fc_case(k, math, out_dt, relu):
    """16 rows of exact data against FC_N rows of weights; the grid's biases. Returns (x, w, bias, expected [16][n])."""
    rng = np.random.default_rng(seed(k, math, out_dt, relu))
    m = dense_magnitude(k)
    x = (rng.integers(-m, m + 1, (16, k)) * 2.0 ** -4).astype(np.float32)
    w = (rng.integers(-m, m + 1, (FC_N, k)) * 2.0 ** -6).astype(np.float32)
    _, gb = grid_table()
    bias = gb[:FC_N] * np.float32(2.0 ** -2)
    check_conv_exact(x.reshape(16, 1, 1, k), w.reshape(FC_N, k, 1, 1), what="fc k %d" % k)
    pre = oracle().conv_f32_nhwc(x.reshape(16, 1, 1, k), w.reshape(FC_N, k, 1, 1), bias, relu=relu,
                                 neg_slope=0.1).reshape(16, FC_N)
    if out_dt == A.HALF:
        tie, _ = f16_ties(pre)
        assert tie.sum() >= 20, "the fc data must reach f16 ties (%d)" % tie.sum()
        want = f16_store(pre)
    else:
        want = pre
    if math == "f16":
        x, w = x.astype(np.float16), w.astype(np.float16)
    return x, w, bias, want


# ------------------------------------------------------------------------------------------------ depthwise
@functools.lru_cache(maxsize=None)
def dw_case(n, h, w, c, r, stride, dil):
    rng = np.random.default_rng(seed(n, h, w, c, r, stride, dil))
    pad = (r - 1) * dil // 2
    x = (rng.integers(-1023, 1024, (n, h, w, c)) * 2.0 ** -8).astype(np.float32)
    wt = (rng.integers(-127, 128, (c, 1, r, r)) * 2.0 ** -6).astype(np.float32)
    bias = rng.uniform(-1, 1, c).astype(np.float32)
    kw = dict(stride=(stride, stride), dil=(dil, dil), pad=(pad, pad))
    # per channel: a 1-channel conv over that channel's taps
    q = conv_quantum(x, wt)
    s = np.stack([conv_f64(np.abs(x[..., j:j + 1]), np.abs(wt[j:j + 1]), **kw)[..., 0] for j in range(c)], -1)
    assert_exact(s, q, "depthwise")
    want = oracle().conv_f32_nhwc(x, wt, bias, group=c, relu=True, neg_slope=0.1, **kw)
    assert (want != np.rint(want)).mean() > 0.5
    return x, wt, bias, want


# ------------------------------------------------------------------------------------------------ f16 average pooling
def pool_tie_planes(n, h, w, c):
    """Channel j alternates f16 values a_j and its f16 successor as a checkerboard: every window of an even tap count
    averages to the exact midpoint, an f16 tie. a_j sweeps both parities, both signs and several binades."""
    j = np.arange(c)
    mag = np.float16(2.0) ** (j % 7 - 3).astype(np.float16)
    base = (mag * (np.float16(1) + np.float16(2.0 ** -10) * (j * 37 % 1024))).astype(np.float16)
    base = np.where((j // 2) % 2 == 1, -base, base).astype(np.float16)
    succ = np.nextafter(base, np.float16(np.inf)).astype(np.float16)
    chk = (np.add.outer(np.arange(h), np.arange(w)) % 2)[None, :, :, None].astype(bool)
    x = np.where(chk, succ[None, None, None, :], base[None, None, None, :])
    return np.broadcast_to(x, (n, h, w, c)).astype(np.float16).copy()
