"""References and designed data for the float kernels that run between the convolutions of FP32 and FP16 nets:
eltwise, activation, scale and softmax (anakin_b200/csrc/pointwise.cu, softmax.cuh), and the error bound of the float
SE gate (se.cu), whose restatement is se_oracle.se_gate_float.

Two kinds of reference:
  * restated kernels: where a kernel's arithmetic is a fixed sequence of fp32 roundings (eltwise, the ReLU kinds of
    activation, scale, the SE gate's pooling order), it is restated op for op in numpy float32 and the results must
    match bit for bit (tests compare uint32 / uint16 views, so that -0 is checked too, and NaN positions);
  * float64 references: where a kernel calls expf or tanhf (sigmoid, tanh, ELU, softmax), the result is compared with
    float64 under a bound derived, in the docstring of each *_bound function, from CUDA's documented maximum errors
    (2 ulp for expf and tanhf; CUDA C++ Programming Guide, Mathematical Functions, single precision) and the
    formula's own fp32 roundings.

Every generator asserts that the edges it was designed for occur. No torch here: this runs on machines without a GPU
(tests/test_cpu_float_ops.py).
"""
import contextlib
import warnings

import numpy as np

import se_oracle as S
from float_exact import f16_ties, seed

F32, F16 = np.float32, np.float16
U = 2.0 ** -24                 # fp32 unit roundoff
FLT_MIN = 2.0 ** -126
ELT_PROD, ELT_SUM, ELT_MAX = 1, 2, 3
ACT_SIGMOID, ACT_RELU, ACT_TANH, ACT_CLIPPED_RELU, ACT_ELU = 1, 2, 3, 4, 5
SOFTMAX_THREADS = 256          # softmax.cuh: one CTA per row, thread t owns t, t + 256, ...


def gamma(k):
    """Relative error bound of k successive fp32 roundings: k u / (1 - k u)."""
    k = np.asarray(k, np.float64)
    return k * U / (1 - k * U)


@contextlib.contextmanager
def _quiet():
    """Overflow, underflow and NaN are the point of the designed data: no warnings for them."""
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        yield


def same_bits(got, want):
    """(mismatch mask) of two float arrays of one dtype: bits must be equal, except that NaN matches NaN of any
    payload (the GPU returns its canonical NaN, numpy propagates the operand's)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    ut = np.uint32 if got.dtype == F32 else np.uint16
    gn, wn = np.isnan(got), np.isnan(want)
    return (gn != wn) | (~gn & (got.view(ut) != want.view(ut)))


def assert_same_bits(got, want, what=""):
    bad = same_bits(got, want)
    if bad.any():
        i = np.flatnonzero(bad.ravel())[:8]
        raise AssertionError("%s: %d of %d differ, first at %s: got %s want %s" % (
            what, int(bad.sum()), bad.size, i.tolist(), np.asarray(got).ravel()[i].tolist(),
            np.asarray(want).ravel()[i].tolist()))


# ------------------------------------------------------------------------------------------------ eltwise
def relu_f32(r):
    """fmaxf(r, 0.f): PTX max.f32 orders -0 below +0 and returns the number when one operand is NaN, so -0 and NaN
    both become +0 (np.maximum would keep -0 and NaN)."""
    r = np.asarray(r, F32)
    return np.where(r > 0, r, F32(0)).astype(F32)


def eltwise(a, b, op, c0=1.0, c1=1.0, relu=False):
    """elt_op in fp32: SUM = __fadd_rn(__fmul_rn(c0, a), __fmul_rn(c1, b)), PROD = __fmul_rn(a, b), MAX = a > b ? a : b;
    then fmaxf(r, 0) with relu. f16 operands are widened exactly and the result rounded once to nearest even."""
    half = np.asarray(a).dtype == F16
    with _quiet():
        x, y = np.asarray(a).astype(F32), np.asarray(b).astype(F32)
        if op == ELT_SUM:
            r = (F32(c0) * x) + (F32(c1) * y)
        elif op == ELT_PROD:
            r = x * y
        else:
            r = np.where(x > y, x, y)
        r = r.astype(F32)
        if relu:
            r = relu_f32(r)
        return r.astype(F16) if half else r


def eltwise_edge_block(dt):
    """Designed (a, b) pairs for ops SUM (c0 = c1 = 1), PROD and MAX, of dtype F16 or F32:
      * f16 ties of both parities: v + ulp(v)/2 and v - ulp(v)/2 for SUM, v * {1.5, 2.5, 0.75, 1.25, 3} for PROD;
      * sums and products past 65504 (65504 + 15 stays, 65504 + 16 = 65520 is a tie that rounds to inf);
      * subnormal operands and results: f16 subnormal sums, 2^-12 * 2^-12 = 2^-24, 2^-13 * 2^-12 = 2^-25 (a tie
        to 0), 3 * 2^-26 (rounds up to 2^-24); fp32 subnormals and 2^-70 * 2^-70 for the fp32 kernel;
      * signed zeros: -0 * 5 = -0, (-0) + (-0) = -0, max(-0, -0) = -0, 0 * -1 = -0: through the relu they become +0;
      * NaN and infinities: inf * 0, inf + -inf, NaN operands.
    The tail is seeded uniform data of both signs."""
    rng = np.random.default_rng(seed("eltwise", dt.__name__))
    m = rng.integers(0, 1024, 256)
    e = rng.integers(-10, 14, 256)
    v = ((1024 + m) * 2.0 ** (e - 10)).astype(np.float64)          # normal f16 values, both mantissa parities
    ulp = 2.0 ** (e - 10)
    sg = np.where(rng.integers(0, 2, 256) == 0, -1.0, 1.0)
    a = [sg * v, sg * v]
    b = [sg * ulp / 2, -sg * ulp / 2]
    a.append(sg * v)
    b.append(np.array([1.5, 2.5, 0.75, 1.25, 3.0])[rng.integers(0, 5, 256)])
    a.append(np.array([65504.0, 65504.0, 65504, 60000, -65504, 300, 256, 4096]))
    b.append(np.array([15.0, 16.0, 65504, 10000, -16, 300, 256, 16]))
    sub = 2.0 ** -24
    a.append(np.array([sub, 3 * sub, -5 * sub, 1023 * sub, 2.0 ** -12, 2.0 ** -13, 3 * 2.0 ** -13, 2.0 ** -14, sub]))
    b.append(np.array([sub, -sub, 2 * sub, sub, 2.0 ** -12, 2.0 ** -12, 2.0 ** -13, -1023 * sub, 0.5]))
    a.append(np.array([-0.0, -0.0, -0.0, 0.0, -0.0, -1.0, 0.0, -3.0]))
    b.append(np.array([5.0, -0.0, 0.0, -1.0, -7.0, -0.0, -0.0, 3.0]))
    a.append(np.array([np.inf, np.inf, -np.inf, np.nan, 1.0, np.inf]))
    b.append(np.array([0.0, -np.inf, 2.0, 1.0, np.nan, 1.0]))
    if dt == F32:
        a.append(np.array([2.0 ** -70, 2.0 ** -140, -(2.0 ** -149), 2.0 ** -126, 3.4e38, 3.4e38, 1.0 + 2.0 ** -23]))
        b.append(np.array([2.0 ** -70, 2.0 ** -9, 2.0 ** -149, -(2.0 ** -127), 3.4e38, 2.0, 1.0 + 2.0 ** -23]))
    a, b = np.concatenate(a), np.concatenate(b)
    tail = 64
    a = np.concatenate([a, rng.uniform(-100, 100, tail)])
    b = np.concatenate([b, rng.uniform(-100, 100, tail)])
    with _quiet():
        return a.astype(dt), b.astype(dt)


def eltwise_data(dt, count):
    """count elements: the edge block, repeated and cut to count (small counts take its first elements)."""
    a, b = eltwise_edge_block(dt)
    reps = -(-count // a.size)
    return np.tile(a, reps)[:count].copy(), np.tile(b, reps)[:count].copy()


def assert_eltwise_edges(dt):
    """What eltwise_edge_block was designed to reach, judged on the restated results."""
    a, b = eltwise_edge_block(dt)
    s, p, m = eltwise(a, b, ELT_SUM), eltwise(a, b, ELT_PROD), eltwise(a, b, ELT_MAX)
    with _quiet():
        pre_s = (a.astype(F32) + b.astype(F32)).astype(F32)
        pre_p = (a.astype(F32) * b.astype(F32)).astype(F32)
    neg0 = lambda r: (r == 0) & np.signbit(r)
    for name, r in (("sum", s), ("prod", p), ("max", m)):
        assert neg0(r).any(), "%s: no -0 result for the relu to turn into +0" % name
    assert np.isnan(s).any() and np.isnan(p).any() and np.isnan(m).any()
    if dt == F16:
        for name, pre in (("sum", pre_s), ("prod", pre_p)):
            tie, up = f16_ties(pre)
            for sgn in (-1, 1):
                for u in (False, True):
                    n = int((tie & (np.sign(pre) == sgn) & (up == u)).sum())
                    assert n >= 10, "%s: %d f16 ties of sign %d rounding %s" % (name, n, sgn, "up" if u else "down")
        assert (np.isinf(s) & np.isfinite(a) & np.isfinite(b)).any(), "no finite sum overflows to inf"
        assert (s == F16(65504)).any() and (pre_s.astype(np.float64) > 65504).any()
        assert (np.isinf(p) & np.isfinite(a) & np.isfinite(b)).any(), "no finite product overflows to inf"
        fsub = lambda r: np.isfinite(r) & (r != 0) & (np.abs(r.astype(np.float64)) < 2.0 ** -14)
        assert fsub(a).any() and fsub(s).any() and fsub(p).any(), "subnormal operands or results missing"
        assert ((pre_p != 0) & (p == 0)).any(), "no product underflows to 0"
        assert f16_ties(pre_p)[0][(np.abs(pre_p) < 2.0 ** -14)].any(), "no subnormal product tie"
    else:
        fsub = lambda r: np.isfinite(r) & (r != 0) & (np.abs(r.astype(np.float64)) < FLT_MIN)
        assert fsub(a).any() and fsub(s).any() and fsub(p).any()
        assert (np.isinf(s) & np.isfinite(a) & np.isfinite(b)).any()


# ------------------------------------------------------------------------------------------------ activation
def relu_kinds(x, act, slope=0.0, coef=1.0):
    """act_op's exact kinds in fp32: RELU = x > 0 ? x : __fmul_rn(x, slope) (so a negative x gives -0 at slope 0, and
    -inf * 0 is NaN); CLIPPED_RELU = min(x > 0 ? x : 0, coef) by compares (NaN -> 0). f16 in: widened, rounded once."""
    half = np.asarray(x).dtype == F16
    with _quiet():
        v = np.asarray(x).astype(F32)
        if act == ACT_RELU:
            y = np.where(v > 0, v, (v * F32(slope)).astype(F32))
        elif act == ACT_CLIPPED_RELU:
            y = np.where(v > 0, v, F32(0))
            y = np.where(y < F32(coef), y, F32(coef))
        else:
            raise ValueError(act)
        y = y.astype(F32)
        return y.astype(F16) if half else y


def act_f64(x, act, coef=1.0):
    """The float64 values that sigmoid / tanh / ELU approximate (the kernel's formulas, evaluated exactly enough)."""
    with _quiet():
        v = np.asarray(x).astype(np.float64)
        if act == ACT_SIGMOID:
            return 1.0 / (1.0 + np.exp(-v))
        if act == ACT_TANH:
            return np.tanh(v)
        if act == ACT_ELU:
            return np.where(v > 0, v, np.float64(F32(coef)) * np.expm1(v))
        raise ValueError(act)


def act_bound(x, act, coef=1.0):
    """|kernel - act_f64| bound for one fp32 result (before any f16 store), from CUDA's 2-ulp expf / tanhf:
      * sigmoid = __fdiv_rn(1, expf(-x) + 1): e = expf(-x) carries 2 ulp <= 2^-22 relative, which reaches
        1 / (1 + e) scaled by e / (1 + e) < 1; the add and the division round once each (2^-24 each). So
        |dy| <= 1.5 * 2^-22 |y|, plus 2^-148 for subnormal roundings. Below FLT_MIN the bound is absolute: once expf
        overflows (x < -88.7) the kernel returns 1 / inf = 0, where the true value is below 2.7e-39.
      * tanh = tanhf(x): 2 ulp, i.e. <= 2^-22 |y|, plus 2 subnormal ulps (2^-148) for tiny x.
      * ELU = x > 0 ? x : __fmul_rn(coef, expf(x) - 1): for x <= 0, e = expf(x) <= 1 carries 2 ulp <= 2^-22 e;
        e - 1 is exact for e >= 1/2 (Sterbenz) and rounds by at most 2^-25 below; the product rounds by 2^-24 |y|.
        The absolute term is what stays near 0, where e - 1 cancels (the reference's formula, kept as it is).
    Second-order terms are covered by a factor 1 + 2^-20, and the float64 evaluation by 2^-48 |y|."""
    y = act_f64(x, act, coef)
    ay = np.abs(y)
    with _quiet():
        if act == ACT_SIGMOID:
            b = 1.5 * 2.0 ** -22 * ay + 2.0 ** -148
            b = np.where(ay < FLT_MIN, np.maximum(b, FLT_MIN), b)
        elif act == ACT_TANH:
            b = 2.0 ** -22 * ay + 2.0 ** -148
        else:
            e = np.exp(np.minimum(np.asarray(x).astype(np.float64), 0))
            b = abs(float(F32(coef))) * (2.0 ** -22 * e + np.where(e < 0.5, 2.0 ** -25, 0.0)) + U * ay + 2.0 ** -149
            b = np.where(np.asarray(x).astype(np.float64) > 0, 0.0, b)
        return np.where(np.isfinite(y), b * (1 + 2.0 ** -20) + 2.0 ** -48 * ay, 0.0)


def check_act_f32(got, x, act, coef=1.0):
    """(max |got - y| / bound, mask of elements past the bound). Infinite and NaN references must be matched exactly."""
    y = act_f64(x, act, coef)
    b = act_bound(x, act, coef)
    g = np.asarray(got, np.float64)
    with _quiet():
        err = np.where(np.isfinite(y), np.abs(g - y), 0.0)
        bad = (np.isfinite(y) & ~(err <= b)) | (np.isnan(y) != np.isnan(g)) | (np.isinf(y) & (g != y))
        ratio = np.where(b > 0, err / np.where(b > 0, b, 1), np.where(err > 0, np.inf, 0))
    return float(ratio.max()), bad


def f16_ordinal(h):
    """f16 values as integers that count f16 numbers: adjacent values differ by 1, -0 and +0 are both 0."""
    b = np.asarray(h, F16).view(np.uint16).astype(np.int32)
    return np.where(b & 0x8000, -(b & 0x7FFF), b)


def check_act_f16(got, x, act, coef=1.0):
    """f16 results against the correctly rounded f16 of the float64 value y. The fp32 intermediate lies within
    act_bound of y, and the f16 store is monotonic, so the kernel's f16 must lie in [rn16(y - b), rn16(y + b)].
    Where both ends are the same f16 number the result is exact. Elsewhere the intermediate lies within its bound of an
    f16 rounding boundary ("near"): when the interval holds two f16 numbers the result may be 1 ulp off the correctly
    rounded one; when it holds more ("wide": the bound is larger than an f16 ulp, as where ELU's expf(x) - 1 cancels)
    it may be further off. Returns (bad, near, wide, off) masks; off: differs from the correctly rounded f16."""
    y = act_f64(x, act, coef)
    b = act_bound(x, act, coef)
    with _quiet():
        want = y.astype(F16)
        lo, hi = (y - b).astype(F16), (y + b).astype(F16)
        g = np.asarray(got, F16)
        fin = np.isfinite(y)
        near = fin & (lo != hi)
        wide = near & (f16_ordinal(hi) - f16_ordinal(lo) >= 2)
        off = same_bits(g, want)
        inside = (g.astype(np.float64) >= lo.astype(np.float64)) & (g.astype(np.float64) <= hi.astype(np.float64))
        bad = np.where(near, ~inside, off)
    return bad, near, wide, off


def all_f16_codes():
    return np.arange(65536, dtype=np.uint32).astype(np.uint16).view(F16)


def f32_activation_grid():
    """fp32 inputs: +-0, subnormals, FLT_MIN, +-FLT_MAX, +-inf, NaN, a log-spaced sweep of both signs from 2^-30 to
    2^20, sigmoid's expf overflow band |x| in [80, 110], tanh's saturation (|x| in [8, 20]), and fp32 neighbours of
    0 and 1."""
    rng = np.random.default_rng(seed("act_f32"))
    with _quiet():
        sweep = 2.0 ** np.linspace(-30, 20, 20001)
        band = np.linspace(80, 110, 6001)
        sat = np.linspace(8, 20, 2001)
        small = np.linspace(-2, 2, 8001)
        special = np.array([0.0, 2.0 ** -149, 3 * 2.0 ** -149, 2.0 ** -130, FLT_MIN, 3.4028234663852886e38, np.inf,
                            1.0, 2.0 ** -24, 2.0 ** -12, 88.72, 88.73, 87.3, 103.9, 104.0])
        pos = np.concatenate([sweep, band, sat, special, rng.uniform(0, 12, 2000)])
        x = np.concatenate([pos, -pos, [np.nan], np.abs(small) * np.sign(small)]).astype(F32)
        x = np.concatenate([x, np.nextafter(F32(1), F32(0))[None], np.nextafter(F32(0), F32(1))[None],
                            np.float32([-0.0])])
    return x


def assert_activation_f32_edges(x):
    v = np.asarray(x, np.float64)
    assert ((v == 0) & np.signbit(v)).any() and ((v == 0) & ~np.signbit(v)).any(), "+-0"
    assert ((np.abs(v) < FLT_MIN) & (v != 0) & (v > 0)).any() and ((np.abs(v) < FLT_MIN) & (v < 0)).any(), "subnormals"
    assert (v == np.float64(np.finfo(F32).max)).any() and (v == -np.float64(np.finfo(F32).max)).any(), "FLT_MAX"
    assert np.isposinf(v).any() and np.isneginf(v).any() and np.isnan(v).any()
    band = (np.abs(v) >= 80) & (np.abs(v) <= 110)
    assert (band & (v < -88.8)).sum() > 1000 and (band & (v > -88.7) & (v < 0)).sum() > 100, "sigmoid's overflow band"
    assert ((np.abs(v) >= 9) & (np.abs(v) <= 20)).sum() > 1000, "tanh's saturation"
    with _quiet():
        assert (act_f64(x, ACT_SIGMOID) < FLT_MIN).sum() > 1000, "sigmoid results below FLT_MIN"
        assert ((v < 0) & (v > -2.0 ** -10)).sum() > 1000, "ELU's cancellation near 0"


# ------------------------------------------------------------------------------------------------ scale
def scale(x, w, b=None):
    """y = __fmul_rn(x, w[c]) [then __fadd_rn(., b[c])] over x [..., c]; f16 widened, one f16 store."""
    half = np.asarray(x).dtype == F16
    with _quiet():
        v = np.asarray(x).astype(F32)
        y = (v * np.asarray(w, F32)).astype(F32)
        if b is not None:
            y = (y + np.asarray(b, F32)).astype(F32)
        return y.astype(F16) if half else y


def scale_data(dt, pixels, c, c_stored):
    """x [pixels, c_stored], w / b [c_stored] (zero in the padding channels, as the Scale op builds them, and the padding
    of x holds values, so that x * 0 + 0 is checked). Designed rows: f16 ties and overflow after the multiply, signed
    zeros and subnormals; the rest seeded uniform of both signs."""
    rng = np.random.default_rng(seed("scale", dt.__name__, pixels, c, c_stored))
    w = rng.uniform(0.25, 4, c_stored) * np.where(rng.integers(0, 2, c_stored) == 0, -1, 1)
    w[: min(c, 3)] = [1.5, -0.75, 2.5][: min(c, 3)]
    b = rng.uniform(-2, 2, c_stored)
    w[c:] = 0
    b[c:] = 0
    x = rng.uniform(-8, 8, (pixels, c_stored))
    rows = min(pixels, 16)
    m = rng.integers(0, 1024, (rows, c_stored))
    e = rng.integers(-16, 14, (rows, c_stored))
    x[:rows] = (1024 + m) * 2.0 ** (e - 10) * np.where(rng.integers(0, 2, (rows, c_stored)) == 0, -1, 1)
    assert pixels >= rows + 3
    x[rows, :] = -0.0
    x[rows + 1, : min(c, 3)] = [40000.0, -50000.0, 30000.0][: min(c, 3)]
    x[rows + 2, :] = 2.0 ** -24 * rng.integers(-1023, 1024, c_stored)
    w, b = w.astype(F32), b.astype(F32)
    with _quiet():
        return x.astype(dt), w, b


def assert_scale_edges(x, w, b, c):
    y = scale(x, w, b)
    yn = scale(x, w)
    assert ((yn == 0) & np.signbit(yn)).any(), "no -0 product"
    if np.asarray(x).dtype == F16:
        with _quiet():
            pre = (x.astype(F32) * w).astype(F32)
        assert f16_ties(pre)[0].sum() >= 4, "no f16 ties after the multiply"
        assert np.isinf(yn).any(), "no product past 65504"
    assert (y[:, c:] == 0).all(), "padding channels must give 0"


# ------------------------------------------------------------------------------------------------ softmax
def softmax_f64(x, axis=-1):
    """Softmax in float64 (max subtracted first), -inf entries giving 0."""
    v = np.asarray(x, np.float64)
    with _quiet():
        m = v.max(axis=axis, keepdims=True)
        e = np.exp(v - m)
        return e / e.sum(axis=axis, keepdims=True)


def softmax_bound(x, adds, axis=-1):
    """|kernel - softmax_f64| bound per element of an fp32 softmax computed as e_i = expf(x_i - max), S = sum e_i,
    y_i = __fdiv_rn(e_i, S):
      * x_i - max rounds with relative error <= 2^-24, which multiplies e_i by exp(d_i * 2^-24): <= |d_i| 2^-24;
      * expf: 2 ulp, <= 2^-22 relative for a normal result; 2^-148 absolute below FLT_MIN;
      * S: every term passes through at most `adds` fp32 additions (rows kernel: ceil(len / 256) per thread, 5
        shuffle levels, 7 cross-warp adds; strided kernel: len sequential adds), all terms positive: gamma(adds);
        the terms' own errors reach S weighted by e_j / S;
      * the final division: 2^-24.
    So |dy_i| <= y_i (eps_i + sum_j y_j eps_j + gamma(adds) + 2^-24) + (len 2^-148) / S, with eps_i the first two
    items, times 1 + 2^-20 for second-order terms, and 2^-149 for a subnormal quotient."""
    v = np.asarray(x, np.float64)
    with _quiet():
        m = v.max(axis=axis, keepdims=True)
        d = v - m
        y = softmax_f64(v, axis)
        e = np.exp(d)
        S = e.sum(axis=axis, keepdims=True)
        eps = np.where(np.isfinite(d), np.abs(d) * U + 2.0 ** -22, 0.0)
        eps_s = (y * eps).sum(axis=axis, keepdims=True)
        n = v.shape[axis]
        b = y * (eps + eps_s + gamma(adds) + U) + n * 2.0 ** -148 / S
        return b * (1 + 2.0 ** -20) + 2.0 ** -149


def rows_adds(length):
    return -(-length // SOFTMAX_THREADS) + 5 + 7


def softmax_exact_rows():
    """Rows whose softmax is exact in fp32, as (x, want) lists:
      * L equal logits at L = 1, 2, 64, 256, 1024, 4096: expf(0) = 1 exactly, the sum is the integer L, 1/L is exact;
      * one logit 105 above the rest: e^-105 lies below half the smallest fp32 subnormal, so the others are +0 and
        the sum is exactly 1;
      * -inf entries: expf(-inf) = +0 exactly, and the finite entries share 1 as above (two equal maxima: 0.5 each)."""
    rows = []
    for n in (1, 2, 64, 256, 1024, 4096):
        v = np.full(n, 3.25, F32)
        rows.append((v, np.full(n, 1.0 / n, F32)))
    for n in (1000, 257):
        v = np.linspace(-5, 5, n).astype(F32)
        v[n // 3] = F32(110.0)
        want = np.zeros(n, F32)
        want[n // 3] = 1
        rows.append((v, want))
    v = np.full(300, -np.inf, F32)
    v[7], v[250] = 2.5, 2.5
    want = np.zeros(300, F32)
    want[7] = want[250] = 0.5
    rows.append((v, want))
    return rows


def softmax_bounded_rows(length):
    """Seeded logits in [-10, 10] with designed entries: a -inf, a logit 30 below the rest's minimum (tiny but normal
    e), and exact duplicates of the maximum; a second row offset by +1e30 and a third by -1e30 in fp32 (without the max
    subtraction expf overflows, or every e is 0), where only the fp32 spacing of 1e30 separates the logits."""
    rng = np.random.default_rng(seed("softmax", length))
    a = rng.uniform(-10, 10, length)
    if length >= 4:
        a[1] = -np.inf
        a[2] = -40.0
        a[3] = a[4:].max()
    big = F32(1e30)
    sp = np.spacing(big)
    k = rng.integers(0, 4, length).astype(np.float64)
    hi = (np.float64(big) + k * np.float64(sp)).astype(F32)
    lo = (-np.float64(big) - k * np.float64(sp)).astype(F32)
    return np.stack([a.astype(F32), hi, lo])


SOFTMAX_LENGTHS = [255, 256, 257, 511, 1000, 4097, 21843]


# ------------------------------------------------------------------------------------------------ SE gate bound
def se_gate_bound(x, ld, w1, b1, w2, b2):
    """|se_oracle.se_gate_float - se_gate_f64| bound per (n, c), propagated in float64 from the fp32 roundings:
      * mean: each pixel passes through se_mean_depth additions, then one division: gamma(depth) sum|x| / hw
        + u |m|;
      * hidden (relu is 1-Lipschitz): sum_c |W1| dm_c + gamma(ceil(c / 32) + 7) (sum_c |W1 m| + |b1|) -- products,
        the lane's sequential sum, 5 butterfly levels and the bias;
      * z: sum_k |W2| dh_k + gamma(r + 2) (sum_k |W2 h| + |b2|);
      * gate: |dz| / 4 (the sigmoid's slope is at most 1/4) plus the explicit sigmoid's own error, 2.25 ulp measured
        over a dense sweep (tests/test_cpu_se.py), taken as 3 * 2^-23 * g.
    Second-order terms: a factor 1.01."""
    n, h, w, c = x.shape
    hw = h * w
    xf = np.asarray(x).astype(np.float64).reshape(n, hw, c)
    W1, W2 = np.asarray(w1, np.float64), np.asarray(w2, np.float64)
    B1, B2 = np.asarray(b1, np.float64), np.asarray(b2, np.float64)
    r = W1.shape[0]
    m = xf.mean(axis=1)
    dm = gamma(S.se_mean_depth(hw, ld, np.asarray(x).dtype.itemsize)) * np.abs(xf).sum(axis=1) / hw + U * np.abs(m)
    pre = m @ W1.T + B1
    hid = np.maximum(pre, 0)
    dh = dm @ np.abs(W1).T + gamma(-(-c // 32) + 7) * (np.abs(m) @ np.abs(W1).T + np.abs(B1))
    z = hid @ W2.T + B2
    dz = dh @ np.abs(W2).T + gamma(r + 2) * (hid @ np.abs(W2).T + np.abs(B2))
    g = 1.0 / (1.0 + np.exp(-z))
    return 1.01 * (dz / 4 + 3 * 2.0 ** -23 * g)
