"""Designed data and expected outputs for replaying the recorded conv plans (tests/golden/conv_plans.json.gz) bit for bit
at the nets' own shapes (tests/test_conv_plan_gpu.py), and what the replay must reach (tests/test_cpu_plan_replay.py).

One data family per math kind, made once per shape and shared by every record of that shape:
- int8: full-range u8 activations and s8 weights, an s8 residual; per-channel bias and scale set from the spread of the
  accumulators, so that the u8 outputs saturate at both ends and most land in range. Expected: the VNNI oracle (the
  same arithmetic as the plain x86 oracle, bit for bit) and its int8 max pooling.
- f16: dense integers times powers of two (float_exact.dense_case's design). Expected: the oracle's fp32 epilogue
  restated on the exact float64 accumulator, (acc + sum_scale * res) + bias and relu / neg_slope, each rounded to fp32,
  then the f16 or fp32 store.
- tf32x3: split operands (float_exact.x3_data's design): every activation has a low part and the sparse weights hit
  every reduction position, so a dropped Alo Whi or Ahi Wlo term changes the bits. Expected: the same epilogue on the
  exact three-term accumulator.

Every generator checks its exactness bound analytically (bound_units) before it draws; the whole-tensor oracle
cross-checks are left to the small shapes of tests/test_cpu_plan_replay.py, which pin the fast references here to
oracle.conv_f32_nhwc and the plain conv_s8_nhwc_x86.

No torch here: the generators run on machines without a GPU.
"""
import collections
import gzip
import json
import os

import numpy as np

import float_exact as F
from anakin_b200 import saber_abi as A

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_plans.json.gz")
SHAPE_FIELDS = ("n", "h", "w", "c", "k", "r", "s", "stride_h", "pad_h", "fuse_pool")
KINDS = {A.MATH_I8: "int8", A.MATH_F16: "f16", A.MATH_TF32X3: "tf32x3"}
FAMILY = {"int8": "int8", "f16": "dense", "tf32x3": "x3"}
X3_RES_MAX = 2048                   # |residual| of the split-term data, in quanta of its products
I8_OUT_SPREAD = 128.0               # the u8 outputs' spread: (acc + bias) * scale has about this standard deviation


def records():
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


def shape_of(desc):
    return tuple(desc[f] for f in SHAPE_FIELDS)


def kind_of(rec):
    return KINDS[rec["desc"]["math"]]


def label(rec):
    return "%s %s" % (rec["case"], json.dumps(rec["env"], sort_keys=True)) if rec["env"] else rec["case"]


def replay_groups(recs=None):
    """{shape: [every successful record of that shape]}, in the order of the records."""
    groups = collections.OrderedDict()
    for rec in records() if recs is None else recs:
        if rec["status"] == A.SUCCESS:
            groups.setdefault(shape_of(rec["desc"]), []).append(rec)
    return groups


def group_id(recs):
    """A readable id from the first record's label without its math kind: resnet50-res4_branch2b-n32."""
    words = [w for w in recs[0]["case"].split() if w not in FAMILY]
    return "-".join(words).replace("->", "to")


def kernel_of(rec):
    return "slab" if rec["slab"] else ("persistent" if rec["persistent"] else "tile")


def reached(recs):
    """{math kind: the set of features the records reach}: kernels, tile widths, splits, fused pools, residuals on tile
    and walker plans, and inner products whose rows are ragged against every row tile."""
    got = collections.defaultdict(set)
    for rec in recs:
        d, kind = rec["desc"], kind_of(rec)
        kernel = kernel_of(rec)
        got[kind].add(kernel)
        if kernel == "tile":
            got[kind].add("tile%d" % rec["block_n"])
            if rec["split"] > 1:
                got[kind].add("split%d" % rec["split"])
        if kernel == "slab":
            got[kind].add("slab+pool" if d["fuse_pool"] else "slab-pool")
        if d["res_dtype"] >= 0 and kernel != "slab":
            got[kind].add(kernel + "+res")
        if d["h"] == 1 and d["w"] == 1 and d["n"] % 128:
            got[kind].add("ragged-fc")
    return got


# ------------------------------------------------------------------------------------------------ geometry
def out_hw(desc):
    oh = (desc["h"] + 2 * desc["pad_h"] - desc["dil_h"] * (desc["r"] - 1) - 1) // desc["stride_h"] + 1
    ow = (desc["w"] + 2 * desc["pad_w"] - desc["dil_w"] * (desc["s"] - 1) - 1) // desc["stride_w"] + 1
    return oh, ow


def conv_kw(desc):
    return dict(stride=(desc["stride_h"], desc["stride_w"]), pad=(desc["pad_h"], desc["pad_w"]),
                dil=(desc["dil_h"], desc["dil_w"]))


def pool_args(desc):
    """(window, pad, stride) of the fused pooling (a stride of 0 means 2, as in the planner)."""
    pk, ps, pp = desc["fuse_pool"], desc["pool_stride"] or 2, desc["pool_pad"]
    return (pk, pk), (pp, pp), (ps, ps)


def reduction(desc):
    return desc["c"] * desc["r"] * desc["s"]


def x3_taps(desc):
    """Nonzero weight taps per output channel: X3_TAPS, or more where k * X3_TAPS does not cover the reduction."""
    return max(F.X3_TAPS, -(-reduction(desc) // desc["k"]))


# ------------------------------------------------------------------------------------------------ exactness bounds
def bound_units(family, desc):
    """The largest |sum| an output can reach, in quanta of the family's products: max|X| max|W| times the taps, plus
    max|residual|. int8: the int32 accumulator's largest |sum|."""
    kk = reduction(desc)
    if family == "int8":
        return kk * 255 * 127
    if family == "dense":
        m = F.dense_magnitude(kk)
        return kk * m * m + F.RES_MAX
    # per tap: Xh Wh 2^10 + Xl Wh + Xh Wl, with Xh, Wh <= 15 and Xl, Wl <= 7
    return x3_taps(desc) * (15 * 15 * 2 ** 10 + 7 * 15 + 15 * 7) + X3_RES_MAX


def assert_bound(family, desc):
    units = bound_units(family, desc)
    limit = 2 ** 31 - 1 if family == "int8" else 2 ** F.EXACT_BITS
    assert units <= limit, "%s %s: sums up to %d quanta are not exact (limit %d)" % (family, shape_of(desc), units,
                                                                                   limit)
    return units


# ------------------------------------------------------------------------------------------------ data
def family_data(family, desc):
    """(x, w, bias, scale) of a shape, in the kind-neutral form: int8 codes, or fp32 values (the f16 kind casts them,
    exactly). The residual comes from residual()."""
    assert_bound(family, desc)
    n, h, w, c, k, r, s = (desc[f] for f in ("n", "h", "w", "c", "k", "r", "s"))
    rng = np.random.default_rng(F.seed(shape_of(desc), family))
    if family == "int8":
        x = rng.integers(0, 256, (n, h, w, c)).astype(np.uint8)
        wt = rng.integers(-127, 128, (k, c, r, s)).astype(np.int8)
        # E[x^2] of uniform codes 0..255, E[w^2] of -127..127: the accumulators' standard deviation
        sigma = np.sqrt(reduction(desc) * (255 * 511 / 6.0) * (127 * 128 / 3.0))
        bias = (rng.uniform(-0.5, 0.5, k) * sigma).astype(np.float32)
        scale = (rng.uniform(0.5, 1.5, k) * (I8_OUT_SPREAD / sigma)).astype(np.float32)
        return x, wt, bias, scale
    if family == "dense":
        m = F.dense_magnitude(reduction(desc))
        x = (rng.integers(-m, m + 1, (n, h, w, c)) * 2.0 ** F.DENSE_EX).astype(np.float32)
        wt = (rng.integers(-m, m + 1, (k, c, r, s)) * 2.0 ** F.DENSE_EW).astype(np.float32)
        return x, wt, rng.uniform(-4, 4, k).astype(np.float32), None      # full 24-bit biases: the + bias rounds
    x = F.split_operand(rng, (n, h, w, c), F.X3_EX, 1)
    wt = F.sparse_weights(rng, k, c, r, s, x3_taps(desc))
    return x, wt, rng.uniform(-1, 1, k).astype(np.float32), None


def residual(family, desc):
    """The residual of a shape (int8 codes or fp32 values exact in f16), or None when the record has none."""
    if desc["res_dtype"] < 0:
        return None
    oh, ow = out_hw(desc)
    shape = (desc["n"], oh, ow, desc["k"])
    rng = np.random.default_rng(F.seed(shape_of(desc), family, "residual"))
    if family == "int8":
        codes = rng.integers(0, 256, shape).astype(np.uint8)        # every code of the residual's 8-bit type
        return codes if desc["res_dtype"] == A.UINT8 else codes.view(np.int8)
    if family == "dense":
        return (rng.integers(-F.RES_MAX, F.RES_MAX + 1, shape) * 2.0 ** (F.DENSE_EX + F.DENSE_EW)).astype(np.float32)
    return (rng.integers(-X3_RES_MAX, X3_RES_MAX + 1, shape) * 2.0 ** (F.X3_EX + F.X3_EW - 10)).astype(np.float32)


def operands(kind, x, w, res, desc):
    """The arrays the kind's plan reads: f16 operands (and a half residual) for the f16 kind."""
    if kind == "f16":
        x, w = x.astype(np.float16), w.astype(np.float16)
    if res is not None and desc["res_dtype"] == A.HALF:
        r16 = res.astype(np.float16)
        assert (r16.astype(np.float32) == res).all(), "the residual must be exact in f16"
        res = r16
    return x, w, res


# ------------------------------------------------------------------------------------------------ references
def accumulator(family, x, w, desc):
    """The exact float64 accumulator of a float family: the dense conv, or the split-term sum
    Ahi Whi + Alo Whi + Ahi Wlo = A Whi + Ahi Wlo (A = Ahi + Alo exactly)."""
    kw = conv_kw(desc)
    if family == "dense":
        return F.conv_f64(x, w, **kw)
    return F.conv_f64(x, F.tf32_hi(w), **kw) + F.conv_f64(F.tf32_hi(x), F.tf32_lo(w), **kw)


def float_epilogue(acc, res, bias, desc):
    """The oracle's fp32 epilogue on an exact accumulator: (acc + sum_scale * res) + bias, then relu / neg_slope, rounded
    to fp32 at each step; the fused max pooling; the store (round half to even for half outputs)."""
    s = acc if res is None else acc + np.float64(desc["sum_scale"]) * res.astype(np.float64)
    v = s.astype(np.float32)                      # exact: the sums are within 2^22 quanta
    v += bias
    if desc["relu"]:
        v = np.where(v > 0, v, v * np.float32(desc["neg_slope"]))
    if desc["fuse_pool"]:
        v = F.oracle().pool_f32(v, *pool_args(desc), A.POOL_MAX, nhwc=True,
                                floor_as_conv=bool(desc["pool_floor_as_conv"]))
    return F.f16_store(v) if desc["out_dtype"] == A.HALF else v


def int8_expected(x, w, bias, scale, res, desc, fast=True):
    o = F.oracle()
    out = o.conv_s8_nhwc_x86(x, w, bias, scale, residual=res, sum_scale=desc["sum_scale"], out_dtype=desc["out_dtype"],
                             relu=bool(desc["relu"]), fast=fast, **conv_kw(desc))
    if desc["fuse_pool"]:
        out = o.pool_s8_nhwc(out, *pool_args(desc), A.POOL_MAX, floor_as_conv=bool(desc["pool_floor_as_conv"]),
                             fast=fast)
    return out


def oracle_expected(kind, x, w, bias, scale, res, desc):
    """The same outputs from the whole-tensor oracle (small shapes only): conv_f32_nhwc, on the three planes
    [Ahi | Alo | Ahi] (*) [Whi | Whi | Wlo] for tf32x3, or the plain conv_s8_nhwc_x86."""
    if kind == "int8":
        return int8_expected(x, w, bias, scale, res, desc, fast=False)
    if kind == "tf32x3":
        x, w = F.x3_expected_operands(x, w)
    o = F.oracle()
    v = o.conv_f32_nhwc(x, w, bias, residual=res, beta=desc["sum_scale"], relu=bool(desc["relu"]),
                        neg_slope=desc["neg_slope"], **conv_kw(desc))
    if desc["fuse_pool"]:
        v = o.pool_f32(v, *pool_args(desc), A.POOL_MAX, nhwc=True, floor_as_conv=bool(desc["pool_floor_as_conv"]))
    return F.f16_store(v) if desc["out_dtype"] == A.HALF else v


def replay(recs):
    """For every record of one shape, in order: (record, (x, w, bias, scale, residual) as its plan reads them, the
    expected output). The data and the accumulators are made once per family, the operands once per kind and residual
    type, and the expected outputs once per descriptor (the switch probes share theirs)."""
    data, ops, wants = {}, {}, {}
    for rec in recs:
        d, kind = rec["desc"], kind_of(rec)
        family = FAMILY[kind]
        if family not in data:
            x, w, bias, scale = family_data(family, d)
            assert_data_coverage(family, x, w, d)
            data[family] = (x, w, bias, scale, None if family == "int8" else accumulator(family, x, w, d))
        x, w, bias, scale, acc = data[family]
        if (kind, d["res_dtype"]) not in ops:
            ops[kind, d["res_dtype"]] = operands(kind, x, w, residual(family, d), d)
        xo, wo, ro = ops[kind, d["res_dtype"]]
        key = json.dumps(d, sort_keys=True)
        if key not in wants:
            if family == "int8":
                want = int8_expected(x, w, bias, scale, ro, d)
            else:
                want = float_epilogue(acc, None if ro is None else ro.astype(np.float32), bias, d)
            assert_output_coverage(kind, want, d)
            wants[key] = want
        yield rec, (xo, wo, bias, scale, ro), wants[key]


# ------------------------------------------------------------------------------------------------ coverage
def assert_data_coverage(family, x, w, desc):
    """What the split-term data must show whatever the outputs: a low part in every activation and in most weight taps,
    and every reduction position hit. (The other families' coverage is in their outputs.)"""
    if family != "x3":
        return
    assert (F.tf32_lo(x) != 0).all(), "every activation must have a low part"
    nz = (w != 0).reshape(w.shape[0], -1)
    assert nz.sum(1).max() <= x3_taps(desc) and nz.any(0).all(), "every reduction position must be hit by some channel"
    assert (F.tf32_lo(w)[w != 0] != 0).mean() > 0.75, "most weight taps must have a low part"


def assert_output_coverage(kind, want, desc):
    """int8 u8 outputs saturate at both ends and a good share lands in range; other outputs are mostly non-integers
    (the + bias and the scale round) and take both signs where no relu clips them."""
    what = "%s %s" % (kind, shape_of(desc))
    if kind == "int8" and desc["out_dtype"] == A.UINT8:
        assert (want == 0).mean() > 0.05 and (want == 255).mean() > 0.001, "%s: the u8 outputs must saturate at both " \
            "ends (%.4f at 0, %.4f at 255)" % (what, (want == 0).mean(), (want == 255).mean())
        assert ((want > 0) & (want < 255)).mean() > 0.3, "%s: too few u8 outputs in range" % what
        return
    v = want.astype(np.float32)
    pos = v[v > 0]
    assert pos.size > 0.1 * v.size and (pos != np.rint(pos)).mean() > 0.5, "%s: the outputs must be mostly " \
        "positive non-integers" % what
    if not desc["relu"]:
        assert (v < 0).mean() > 0.1, "%s: without relu the outputs must take both signs" % what
