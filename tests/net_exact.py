"""Designed weights whose every sum is exact, and an exact walk of the FP32 and FP16 nets.

The float kernels are exact on data whose sums are exact in fp32 (float_exact.py): the result then does not depend on
the accumulation order, the plan, the tile width or split-K, and the only roundings left are `+ bias`, the store and
the AVG division. This module designs whole nets with that property, and walks them in float64, rounding where the
device rounds, so that every edge of a Net can be predicted bit for bit.

Design. Every folded conv / Dense weight is a small integer: each output channel has a few nonzero taps. A conv whose
output goes through a ReLU gets one +1 tap and one or two taps of -1 / -2; the conv that ends a residual block gets only
negative taps, so the block output ReLU(shortcut - sum) stays below the largest shortcut value. Activations are
multiples of the input's quantum, their largest value does not grow from layer to layer, and so every sum stays below
2^22 quanta at any depth. The classifier's taps are +-1. Biases are multiples of the quantum, chosen on image 0 of the
design so that each ReLU clips a part of its channel, and capped so that magnitudes cannot creep up over 100 layers.

The BatchNorm / Scale parameters are chosen backwards from the folded weights:
  * var / factor + eps is a power of 4 in fp32, so 1 / sqrt is exact; var / factor alone is not one, so a fold that
    drops eps changes bits; factor is not 1, so a fold that ignores it changes bits;
  * gamma = +-2^G is large, and the stored weights are the folded ones divided by gamma * 2^m: down among the f16
    subnormals below 2^-24, so rounding them to f16 before the fold (instead of after it) changes bits;
  * mean and beta are multiples of the quantum after the fold.
The input is 12-bit integers times 2^-10, different in every image: the f16 staging of the stem rounds some of them.

The walk groups nodes with oracle/model_walker.plan (independent of the C++ grouping) and asserts, layer by layer, that
every conv, Dense and AVG sum is exact given its actual (rounded) inputs, and that the data is dense: no edge is mostly
zero, every ReLU clips some values but not all, residuals change outputs, images differ, and the FP16 stores round.

No torch here: it runs on machines without a GPU.
"""
import functools

import numpy as np

from float_exact import EXACT_BITS, _tap_slices, assert_exact, conv_f64, f16_store, quantum_of, seed, tf32_hi, tf32_lo

# net: input height / width. The 224 x 224 ResNets and MobileNet-v1 end in a 7 x 7 global average: its division by 49
# leaves full 24-bit mantissas in front of the classifier, whose fp32 sums then round (and the 3xTF32 split of a
# 24-bit value drops bits). At 256 x 256 (Graph.Reshape) the window is 8 x 8 and the division by 64 is exact.
NETS = {"tiny_resnet": 32, "tiny_mobilenet": 32, "resnet50": 256, "resnet101": 256, "vgg16": 224,
        "mobilenet_v1": 256}

IN_EXP = -10            # input quantum
IN_MAX = 3000           # |X| <= 3000: integers of up to 12 bits, so some inputs are not f16 numbers
BIAS_CAP = 64           # the biases of layers without a ReLU, and the BatchNorm means, are at most 64 quanta
BIAS_MAX = 2048         # a bias is at most 2048 quanta: a fixed cap, so that magnitudes do not compound with depth
CLIP_SHARE = 0.3        # a ReLU bias is minus the 30 % quantile of its channel's pre-activation on design image 0
FOLD_G = 26             # gamma * 2^m = 2^26..2^28: stored weights are multiples of 2^-26 and below, f16-inexact
MIN_NONZERO = 0.3       # every compared edge has at least 30 % nonzero values
MIN_F16_ROUNDED = 0.01  # the fp16 walk's conv stores round at least 1 % of their values


def _attr(node, key):
    v = node["attrs"][key]
    return np.asarray(v["tensor"] if isinstance(v, dict) else v, np.float32)


def image(name, i):
    hw = NETS[name]
    rng = np.random.default_rng(seed(name, "image", i))
    return (rng.integers(-IN_MAX, IN_MAX + 1, (3, hw, hw)) * 2.0 ** IN_EXP).astype(np.float32)


def images(name, batch):
    return np.stack([image(name, i) for i in range(batch)])


# ------------------------------------------------------------------------------------------------ conv / pooling
def conv_grouped(x, w, group, stride, pad, dil):
    """conv_f64 for group 1 and for depthwise convolutions (one input channel per group)."""
    if group == 1:
        return conv_f64(x, w, stride, pad, dil)
    n, h, wd, c = x.shape
    assert group == c == w.shape[0] and w.shape[1] == 1, "only plain and depthwise convolutions"
    r, s = w.shape[2:]
    xp = np.zeros((n, h + 2 * pad[0], wd + 2 * pad[1], c), np.float64)
    xp[:, pad[0]:pad[0] + h, pad[1]:pad[1] + wd] = x
    acc = None
    for ky, kx, sl in _tap_slices(n, h, wd, r, s, stride, pad, dil):
        t = xp[sl] * np.asarray(w[:, 0, ky, kx], np.float64)
        acc = t if acc is None else acc + t
    return acc


def pool_out(h, k, s, p, global_pooling):
    """Caffe's ceil-mode output size (the nets use no floor mode)."""
    if global_pooling:
        return 1
    o = -(-(h + 2 * p - k) // s) + 1
    return o - 1 if (o - 1) * s >= h + p else o


def pool_windows(x, a):
    """[(tap array, valid mask)] per tap of a pooling, the taps clipped to the input."""
    n, h, w, c = x.shape
    if a["global_pooling"]:
        return [(x[:, y:y + 1, z:z + 1], None) for y in range(h) for z in range(w)], (h, w)
    (kh, kw), (sh, sw), (ph, pw) = a["pool_size"], a["strides"], a["padding"]
    oh, ow = pool_out(h, kh, sh, ph, False), pool_out(w, kw, sw, pw, False)
    hp, wp = (oh - 1) * sh + kh, (ow - 1) * sw + kw
    xp = np.zeros((n, hp, wp, c), np.float64)
    valid = np.zeros((1, hp, wp, 1), bool)
    xp[:, ph:ph + h, pw:pw + w] = x[:, :hp - ph, :wp - pw]
    valid[:, ph:ph + h, pw:pw + w] = True
    taps = []
    for ky in range(kh):
        for kx in range(kw):
            sl = (slice(None), slice(ky, ky + (oh - 1) * sh + 1, sh), slice(kx, kx + (ow - 1) * sw + 1, sw))
            taps.append((xp[sl], valid[sl]))
    return taps, (kh, kw)


# ------------------------------------------------------------------------------------------------ fold
def fold(g, no_eps=False, f16_first=False):
    """(w, bias) float32 of a conv group, folded as operators.cpp's fold_bn_scale does it, step by step in fp32.
    no_eps / f16_first: the fold without eps, or after rounding the stored weights to f16 (negative controls)."""
    a = g.head["attrs"]
    w = _attr(g.head, "weight_1").copy()
    k = w.shape[0]
    b = _attr(g.head, "weight_2").reshape(-1).copy() if a.get("bias_term") else np.zeros(k, np.float32)
    if f16_first:
        w = f16_store(w).astype(np.float32)
    if g.bn is None and g.scale is None:
        return w, b
    f32 = np.float32
    if g.bn is not None:
        mean = _attr(g.bn, "weight_1").reshape(-1)
        var = _attr(g.bn, "weight_2").reshape(-1)
        factor = f32(_attr(g.bn, "weight_3").reshape(-1)[0])
        eps = f32(g.bn["attrs"]["epsilon"])
    else:
        mean, var, factor, eps = np.zeros(k, f32), np.ones(k, f32), f32(1), f32(0)
    if g.scale is not None:
        gamma = _attr(g.scale, "weight_1").reshape(-1)
        beta_s = _attr(g.scale, "weight_2").reshape(-1) if g.scale["attrs"].get("bias_term") else None
    else:
        gamma, beta_s = np.ones(k, f32), None
    f = f32(1) if factor == 0 else f32(1) / factor
    alpha = var * f if no_eps else var * f + eps
    alpha = f32(1) / np.sqrt(alpha)
    beta = (f32(-1) * (mean * f)) * alpha
    alpha = gamma * alpha
    beta = beta * gamma + beta_s if beta_s is not None else beta * gamma
    return w * alpha[:, None, None, None], b * alpha + beta


# ------------------------------------------------------------------------------------------------ the walk
class Walk:
    """Stored values of every node of a walked net: `vals[node]` (float32 / float16 numpy, NHWC or [n, 1, 1, k]), the
    float64 softmax `prob`, and counters of what the assertions saw."""

    def __init__(self):
        self.vals, self.prob, self.stats = {}, None, {"f16_rounded": 0, "conv_stores": 0, "sums": 0,
                                                       "stem_rounded": 0}


def edge_dtype(graph, precision):
    """{node: np.float16 | np.float32} of every stored edge: an fp16 net stores half unless a real consumer (Split
    passed through) is a Softmax or an Output, or the node is the graph Input (net.cpp, NetCore::init step 2)."""
    nodes = {n["name"]: n for n in graph["nodes"]}

    def real(name):
        for o in nodes[name]["outs"]:
            if nodes[o]["op"] == "Split":
                yield from real(o)
            else:
                yield o
    out = {}
    for n in graph["nodes"]:
        half = precision == "fp16" and n["op"] != "Input" and \
            not any(nodes[c]["op"] in ("Softmax", "Output") for c in real(n["name"]))
        out[n["name"]] = np.float16 if half else np.float32
    return out


def _relu(f, slope):
    return np.where(f > 0, f, (f * np.float32(slope)).astype(np.float32)).astype(np.float32)


def _store(v32, dt):
    return f16_store(v32) if dt == np.float16 else np.asarray(v32, np.float32)


def _check_tf32_split(x, what):
    """3xTF32 multiplies hi(x) and the top 11 bits of lo(x) with the weights: x must have at most 22 bits."""
    x = np.asarray(x, np.float32)
    assert (tf32_hi(x) + tf32_hi(tf32_lo(x)) == x).all(), "%s: an operand has more than 22 significant bits" % what


def _dense_check(w, what):
    w = np.asarray(w, np.float32)
    assert (tf32_lo(w) == 0).all(), "%s: a weight has a nonzero TF32 low plane" % what
    assert (f16_store(w).astype(np.float32) == w).all(), "%s: a weight is not an f16 number" % what


def _exact_sum(abs_sum, quantum, what, stats):
    stats["max_bits"] = max(stats.get("max_bits", 0), float(np.log2(assert_exact(abs_sum, quantum, what))))
    stats["sums"] += int(np.asarray(abs_sum).size)


def walk(graph, x_nchw, precision, mutate=(), check=True):
    """Walk `graph` (modelzoo dict form) on x_nchw in `precision` ("fp32" / "fp16"). `mutate`: negative controls, each
    a bug the GPU comparison must catch (no_eps, f16_before_fold, avg_counts_padding, nhwc_flatten, residual_other,
    swap_tail); a mutated walk skips the exactness and density assertions."""
    from oracle import model_walker as MW
    mutate = set(mutate)
    nodes = {n["name"]: n for n in graph["nodes"]}
    dts = edge_dtype(graph, precision)
    half = precision == "fp16"
    wk = Walk()
    vals, st = wk.vals, wk.stats
    x_in = np.ascontiguousarray(np.transpose(np.asarray(x_nchw, np.float32), (0, 2, 3, 1)))
    n_img = x_in.shape[0]

    def density(name, v, pre=None, relu=False):
        if not check:
            return
        v = np.asarray(v, np.float32)
        assert (v != 0).mean() >= MIN_NONZERO, "%s: only %.2f of the values are nonzero" % (name, (v != 0).mean())
        if relu:
            clip = (np.asarray(pre) < 0).mean()
            assert 0.01 <= clip < 1 - MIN_NONZERO, "%s: the ReLU clips %.3f of the values" % (name, clip)
        for i in range(1, n_img):
            assert not np.array_equal(v[i], v[0]), "%s: image %d equals image 0" % (name, i)

    for g in MW.plan(graph):
        a = g.head["attrs"]
        name = g.head["name"]
        if g.kind == "input":
            vals[name] = x_in
        elif g.kind in ("split", "output"):
            vals[name] = vals[g.inputs[0]]
        elif g.kind == "conv":
            src = vals[g.inputs[0]].astype(np.float32)
            if half and nodes[g.inputs[0]]["op"] == "Input":
                staged = f16_store(src).astype(np.float32)          # the stem converts its fp32 input to f16
                st["stem_rounded"] += int((staged != src).sum())
                src = staged
            w, bias = fold(g, "no_eps" in mutate, "f16_before_fold" in mutate and half)
            if check:
                _dense_check(w, name)
                if not half:
                    _check_tf32_split(src, name + " input")
            if half:
                w = f16_store(w).astype(np.float32)
            kw = dict(stride=tuple(a["strides"]), pad=tuple(a["padding"]), dil=tuple(a["dilation_rate"]))
            grp = int(a["group"])
            acc = conv_grouped(src, w, grp, **kw)
            res = None
            if g.elt is not None:
                res = acc if "residual_other" in mutate else vals[g.residual].astype(np.float64)
            if check:
                s = conv_grouped(np.abs(src.astype(np.float64)), np.abs(w.astype(np.float64)), grp, **kw)
                qx = quantum_of(src)
                q = np.array([qx * quantum_of(w[j]) for j in range(w.shape[0])])
                if res is not None:
                    s = s + np.abs(res)
                    q = np.minimum(q, quantum_of(res))
                _exact_sum(s, q, name, st)
            t = (acc if res is None else acc + res).astype(np.float32)
            if check:
                assert (t.astype(np.float64) == (acc if res is None else acc + res)).all(), name
            f = (t + bias).astype(np.float32)
            if check and res is not None:
                without = (acc.astype(np.float32) + bias).astype(np.float32)
                assert (without != f).mean() > 0.3, "%s: the residual changes only %.2f of the outputs" % (
                    name, (without != f).mean())
            pre = f
            if g.relu:
                f = _relu(f, g.relu_alpha)
            dt = dts[g.out_name]
            out = _store(f, dt)
            if dt == np.float16:
                st["f16_rounded"] += int((out.astype(np.float32) != f).sum())
            st["conv_stores"] += f.size
            density(name, out, pre, g.relu)
            for m in g.nodes:
                vals[m["name"]] = out
        elif g.kind == "pool":
            src = vals[g.inputs[0]].astype(np.float64)
            if "swap_tail" in mutate and a["global_pooling"]:
                src = src[np.r_[n_img - 1, 1:n_img - 1, 0]] if n_img > 1 else src
            taps, (kh, kw) = pool_windows(src, a)
            dt = dts[name]
            if a["method"] == "MAX":
                r = taps[0][0] if taps[0][1] is None else np.where(taps[0][1], taps[0][0], -np.inf)
                for tv, ok in taps[1:]:
                    r = np.maximum(r, tv if ok is None else np.where(ok, tv, -np.inf))
                out = _store(r.astype(np.float32), dt)
            else:
                assert a["method"] == "AVG" and a["global_pooling"] and tuple(a["padding"]) == (0, 0), name
                s = sum(tv for tv, _ in taps)
                if check:
                    _exact_sum(sum(np.abs(tv) for tv, _ in taps), quantum_of(src), name, st)
                d = np.prod(a["pool_size"]) if "avg_counts_padding" in mutate else kh * kw
                out = _store(s.astype(np.float32) / np.float32(d), dt)        # __fdiv_rn
            density(name, out)
            vals[name] = out
        elif g.kind == "dense":
            x = vals[g.inputs[0]].astype(np.float64)
            n = x.shape[0]
            order = (0, 1, 2, 3) if "nhwc_flatten" in mutate else (0, 3, 1, 2)   # Dense flattens NCHW
            xf = np.ascontiguousarray(np.transpose(x, order)).reshape(n, -1)
            wd = _attr(g.head, "weight_1").reshape(int(a["out_dim"]), -1)
            if check:
                _dense_check(wd[wd != 0], name)
            rows, cols = np.nonzero(wd)
            wv = wd[rows, cols].astype(np.float64)
            kout = wd.shape[0]
            acc = np.stack([np.bincount(rows, xf[i, cols] * wv, kout) for i in range(n)])
            if check:
                s = np.stack([np.bincount(rows, np.abs(xf[i, cols] * wv), kout) for i in range(n)])
                _exact_sum(s, quantum_of(xf) * quantum_of(wv), name, st)
            b = _attr(g.head, "weight_2").reshape(-1) if a.get("bias_term") else np.zeros(kout, np.float32)
            f = (acc.astype(np.float32) + b).astype(np.float32)
            out = _store(f, dts[name]).reshape(n, 1, 1, kout)
            density(name, out)
            vals[name] = out
            if g.relu:      # the ReLU after a Dense is an op of its own: it reads the stored values
                rn = g.nodes[-1]["name"]
                r = _relu(out.astype(np.float32), g.relu_alpha)
                vals[rn] = _store(r, dts[rn])
                density(rn, vals[rn], out.astype(np.float32), True)
        elif g.kind == "softmax":
            from float_ops_ref import softmax_f64
            x = vals[g.inputs[0]]
            wk.prob = softmax_f64(x.reshape(x.shape[0], -1).astype(np.float64))
            vals[name] = wk.prob.astype(np.float32).reshape(x.shape)
        else:
            raise NotImplementedError("%s: %s" % (name, g.kind))
    if check and half:
        share = st["f16_rounded"] / st["conv_stores"]
        assert share >= MIN_F16_ROUNDED, "only %.4f of the fp16 conv stores round" % share
        assert st["stem_rounded"] > 0, "the f16 staging of the stem rounds no input"
    return wk


# ------------------------------------------------------------------------------------------------ design
def _pow4_var(t, f, eps):
    """A var with fp32(fp32(var * f) + eps) == t (a power of 4) while var * f is not t itself."""
    f32 = np.float32
    v = f32((np.float64(t) - np.float64(eps)) / np.float64(f))
    for _ in range(64):
        got = f32(f32(v * f) + eps)
        if got == t:
            break
        v = np.nextafter(v, f32(np.inf) if got < t else f32(-np.inf))
    assert f32(f32(v * f) + eps) == t, "no var for 4^%g" % np.log2(t)
    assert f32(v * f) != t
    return v


def _taps(rng, k, kk, kind):
    """[k][kk] small-integer weights of one layer (reduction index as in the KCRS flattening)."""
    w = np.zeros((k, kk), np.float32)
    for j in range(k):
        if kind == "stem":
            pos = rng.choice(kk, 4, replace=False)
            w[j, pos] = rng.choice([-2, -1, 1, 2], 4)
        elif kind == "head":
            pos = rng.choice(kk, 3, replace=False)
            w[j, pos] = rng.choice([-1, 1], 3)
        else:
            nneg = int(rng.integers(1, 3)) if kind == "residual" else 1
            lead = 0 if kind == "residual" else 1
            pos = rng.choice(kk, lead + nneg, replace=False)
            w[j, pos[lead:]] = rng.choice([-2, -1], nneg, p=[0.25, 0.75])
            if lead:
                w[j, pos[0]] = 1
    return w


def _bias(rng, pre, q, relu, cap):
    """Multiples of the quantum q: minus the CLIP_SHARE quantile of each channel's pre-activation for a ReLU layer,
    small random ones otherwise; at most `cap` above zero."""
    k = pre.shape[-1]
    if relu:
        b = np.rint(-np.quantile(pre.reshape(-1, k), CLIP_SHARE, axis=0) / q) * q
    else:
        b = rng.integers(-BIAS_CAP, BIAS_CAP + 1, k) * q
    return np.minimum(b, cap)


def _set(node, key, arr, like=None):
    shape = np.shape(node["attrs"][key]) if like is None else like
    node["attrs"][key] = np.asarray(arr, np.float32).reshape(shape)


def _fold_inverse(rng, g, w_f, b_f, q):
    """Write the conv's stored weights and its BatchNorm / Scale parameters so that fold(g) gives (w_f, b_f)."""
    conv = g.head
    k = w_f.shape[0]
    if g.bn is None and g.scale is None:
        _set(conv, "weight_1", w_f)
        if conv["attrs"].get("bias_term"):
            _set(conv, "weight_2", b_f)
        else:
            assert (b_f == 0).all()
        return
    assert g.bn is not None and g.scale is not None, conv["name"]
    eps = np.float32(g.bn["attrs"]["epsilon"])
    factor = np.float32(rng.choice([0.5, 2.0, 4.0]))
    f = np.float32(1) / factor
    m = rng.integers(1, 9, k)                          # var / factor + eps = 4^-m, 1 / sqrt = 2^m (4^-8 > eps)
    var = np.array([_pow4_var(np.float32(4.0 ** -int(mj)), f, eps) for mj in m], np.float32)
    gexp = FOLD_G - m + rng.integers(0, 3, k)
    sign = rng.choice([-1.0, 1.0], k)
    gamma = sign * 2.0 ** gexp
    alpha = gamma * 2.0 ** m                           # the folded scale, exactly
    mu = rng.integers(-BIAS_CAP, BIAS_CAP + 1, k)
    mean = mu * q * np.float64(factor) / 2.0 ** (m + gexp)      # -(mean / factor) * 2^m * gamma = -sign * mu * q
    beta_s = b_f + sign * mu * q
    raw = w_f / alpha[:, None, None, None]
    if conv["attrs"].get("bias_term"):
        rho = rng.integers(-BIAS_CAP, BIAS_CAP + 1, k)
        _set(conv, "weight_2", rho * q / alpha)
        beta_s = beta_s - rho * q
    _set(conv, "weight_1", raw)
    _set(g.bn, "weight_1", mean)
    _set(g.bn, "weight_2", var)
    _set(g.bn, "weight_3", [factor])
    _set(g.scale, "weight_1", gamma)
    _set(g.scale, "weight_2", beta_s)
    g.scale["attrs"]["bias_term"] = True
    w_got, b_got = fold(g)
    assert np.array_equal(w_got, w_f.astype(np.float32)) and np.array_equal(b_got, b_f.astype(np.float32)), \
        "%s: the fold does not give the designed weights" % conv["name"]
    assert (f16_store(raw).astype(np.float32) != raw)[w_f != 0].mean() > 0.5, \
        "%s: the stored weights must not be f16 numbers" % conv["name"]


@functools.lru_cache(maxsize=None)
def design(name):
    """{node: {attr: float32 array}} of the designed parameters of net `name` (any batch), after walking design image
    0 to choose the biases."""
    from anakin_b200 import modelzoo
    from oracle import model_walker as MW
    graph = modelzoo.build(name, 1, "fp32", centered=False)
    nodes = {n["name"]: n for n in graph["nodes"]}
    rng = np.random.default_rng(seed(name, "design"))
    q = 2.0 ** IN_EXP
    x = images(name, 1)
    vals = {}
    for g in MW.plan(graph):
        a = g.head["attrs"]
        nm = g.head["name"]
        if g.kind == "input":
            vals[nm] = np.transpose(x, (0, 2, 3, 1)).astype(np.float64)
        elif g.kind in ("split", "output", "softmax"):
            vals[nm] = vals[g.inputs[0]]
        elif g.kind == "conv":
            src = vals[g.inputs[0]]
            wt = _attr(g.head, "weight_1")
            k, cpg, r, s = wt.shape
            kind = "stem" if nodes[g.inputs[0]]["op"] == "Input" else \
                "residual" if g.elt is not None else "relu" if g.relu else "linear"
            w_f = _taps(rng, k, cpg * r * s, kind).reshape(k, cpg, r, s)
            kw = dict(stride=tuple(a["strides"]), pad=tuple(a["padding"]), dil=tuple(a["dilation_rate"]))
            pre = conv_grouped(src, w_f, int(a["group"]), **kw)
            if g.elt is not None:
                pre = pre + vals[g.residual]
            b_f = _bias(rng, pre, q, g.relu, BIAS_MAX * q)
            _fold_inverse(rng, g, w_f, b_f, q)
            y = pre + b_f
            if g.relu:
                y = np.maximum(y, 0)
            for m in g.nodes:
                vals[m["name"]] = y
        elif g.kind == "pool":
            src = vals[g.inputs[0]]
            taps, (kh, kw) = pool_windows(src, a)
            if a["method"] == "MAX":
                r = None
                for tv, ok in taps:
                    tv = tv if ok is None else np.where(ok, tv, -np.inf)
                    r = tv if r is None else np.maximum(r, tv)
            else:
                r = sum(tv for tv, _ in taps) / (kh * kw)
            vals[nm] = r
        elif g.kind == "dense":
            src = vals[g.inputs[0]]
            xf = np.transpose(src, (0, 3, 1, 2)).reshape(1, -1)
            kout = int(a["out_dim"])
            kind = "relu" if g.relu else "head"
            wd = _taps(rng, kout, xf.shape[1], kind)
            pre = xf @ wd.T.astype(np.float64)
            qd = quantum_of(xf) if kind == "head" else q
            b = _bias(rng, pre, qd, False, BIAS_MAX * q)      # one row: no quantile to take
            _set(g.head, "weight_1", wd)
            _set(g.head, "weight_2", b)
            y = pre + b
            if g.relu:
                y = np.maximum(y, 0)
            vals[nm] = y.reshape(1, 1, 1, kout)
            for m in g.nodes:
                vals[m["name"]] = vals[nm]
        else:
            raise NotImplementedError(g.kind)
    keys = ("weight_1", "weight_2", "weight_3", "bias_term")
    return {n["name"]: {k: (np.asarray(n["attrs"][k], np.float32) if k != "bias_term" else n["attrs"][k])
                        for k in keys if k in n["attrs"]}
            for n in graph["nodes"] if n["op"] in ("Convolution", "BatchNorm", "Scale", "Dense")}


def designed_graph(name, batch):
    """modelzoo's graph of `name` at `batch` with the designed parameters. Its Input keeps modelzoo's shape: a Net of a
    net whose NETS size differs is reshaped to it (Graph.Reshape)."""
    from anakin_b200 import modelzoo
    graph = modelzoo.build(name, batch, "fp32", centered=False)
    params = design(name)
    for n in graph["nodes"]:
        for k, v in params.get(n["name"], {}).items():
            n["attrs"][k] = v
    return graph


@functools.lru_cache(maxsize=None)
def exact_walk(name, batch, precision):
    """(graph, x, Walk) of the designed net at `batch`, after every assertion of the walk."""
    graph = designed_graph(name, batch)
    x = images(name, batch)
    return graph, x, walk(graph, x, precision)
