"""CPU restatement of the squeeze-and-excitation operators (anakin_b200/csrc/se.cu, contracts in include/b200_saber.h)
and a model walker for SE nets (Axpy, the SE gate, Sigmoid) in FP32 and in INT8 x86 semantics.

The walker follows oracle/model_walker.py op for op -- the same conv, pooling, inner-product and softmax restatements
(oracle/pyoracle.py), the same edge typing -- and adds:
  * the SE gate (global AVE Pooling -> 1x1 Convolution + bias -> ReLU -> 1x1 Convolution + bias -> Sigmoid, read as
    input 0 of an Axpy): an fp32 [n, C] gate in every precision, by se_gate below;
  * Axpy [+ ReLU]: axpy_f32 (fmaf, as the reference's saber_axpy.cu computes once nvcc contracts it) and the INT8 rule
    axpy_q8, which is this project's own (the reference has no INT8 Axpy).
"""
import numpy as np

from oracle import model_walker as W
from oracle import pyoracle as O

DT_FLOAT, DT_INT8, DT_UINT8 = O.DT_FLOAT, O.DT_INT8, O.DT_UINT8
F32 = np.float32


def _bits(u):
    return np.uint32(u).view(np.float32)


# ------------------------------------------------------------------------------------------------ sigmoid
_LOG2E, _C1, _C2 = _bits(0x3fb8aa3b), _bits(0x3f318000), _bits(0xb95e8083)
_POLY = [_bits(0x39500d01), _bits(0x3ab60b61), _bits(0x3c088889), _bits(0x3d2aaaab), _bits(0x3e2aaaab), F32(0.5),
         F32(1.0), F32(1.0)]
_P64 = _bits(0x1f800000)


def sigmoid_f32(z):
    """se.cu's se_sigmoid, op for op in float32: e = exp(-|z|) by Cody-Waite (k = rint(t log2 e), r = t - k C1 - k C2)
    and a degree-7 Horner polynomial, scaled by 2^k; 1 / (1 + e) for z >= 0, e / (1 + e) otherwise."""
    z = np.asarray(z, F32)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        a = np.minimum(np.abs(z), F32(126))
        t = -a
        k = np.rint(t * _LOG2E).astype(F32)
        r = t - k * _C1
        r = r - k * _C2
        q = np.full_like(r, _POLY[0])
        for c in _POLY[1:]:
            q = q * r + c
        ki = k.astype(np.int32)
        normal = ki >= -126
        p_hi = ((np.where(normal, ki, 0) + 127).astype(np.uint32) << 23).view(F32)
        p_lo = ((np.where(normal, 0, ki + 64) + 127).astype(np.uint32) << 23).view(F32)
        e = np.where(normal, q * p_hi, (q * p_lo) * _P64).astype(F32)
        den = F32(1) + e
        return np.where(z >= 0, F32(1) / den, e / den).astype(F32)


# ------------------------------------------------------------------------------------------------ Axpy
def fmaf(a, b, c):
    """float32 fused multiply-add, exactly rounded once: the float64 product is exact, the float64 sum's error is
    recovered by TwoSum and decides the one case a second rounding could get wrong (a sum on a float32 midpoint)."""
    a, b, c = (np.asarray(v, F32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    s = p + c.astype(np.float64)
    bb = s - p
    err = (p - (s - bb)) + (c.astype(np.float64) - bb)
    with np.errstate(over="ignore", invalid="ignore"):
        r = s.astype(F32)
        other = np.nextafter(r, np.where(s > r.astype(np.float64), F32(np.inf), F32(-np.inf)).astype(F32))
        mid = (r.astype(np.float64) + other.astype(np.float64)) / 2 == s
        # on a midpoint both neighbours are at the same distance from s: err picks the side of the true value
        fix = mid & (r != other) & (err != 0)
        r = np.where(fix, np.where(err > 0, np.maximum(r, other), np.minimum(r, other)), r)
    return r.astype(F32)


def axpy_f32(g, x, y, relu=False, neg_slope=0.0, contract=True):
    """g [n, C], x / y [n, h, w, C] fp32: fmaf(g, x, y), then the ReLU with negative slope. contract=False: the product
    and the sum rounded on their own, the reference's axpy_nv_basic as written."""
    gb = np.asarray(g, F32)[:, None, None, :]
    t = fmaf(gb, x, y) if contract else (np.asarray(x, F32) * gb + np.asarray(y, F32)).astype(F32)
    if relu:
        t = np.where(t > 0, t, t * F32(neg_slope)).astype(F32)
    return t


def axpy_f16(g, x, y, relu=False, neg_slope=0.0):
    """The fp32 rule on the widened f16 operands, one round-half-even store."""
    return axpy_f32(g, np.asarray(x, np.float16).astype(F32), np.asarray(y, np.float16).astype(F32), relu,
                    neg_slope).astype(np.float16)


def axpy_factors(sx, x_dt, sy, y_dt, so, out_dt):
    """(ax, ay) of the INT8 rule: f = scale * (127/255 for u8), ax = f_x / f_out, ay = f_y / f_out (fp32 steps, with the
    u8 factor the float division 127 / 255 as the INT8 eltwise computes it)."""
    u = F32(127) / F32(255)

    def f(s, dt):
        return F32(s) * (u if dt == DT_UINT8 else F32(1))
    fo = f(so, out_dt)
    return F32(f(sx, x_dt) / fo), F32(f(sy, y_dt) / fo)


def axpy_q8(g, qx, qy, ax, ay, out_dt, relu=False):
    """INT8 Axpy: t = (g * ax) * qx + qy * ay, each product and the sum rounded to fp32 on its own (no FMA); ReLU
    max(t, 0); round half to even and saturate to the output's 8-bit range. g [n, C] fp32; qx, qy [n, h, w, C] codes."""
    gs = (np.asarray(g, F32) * F32(ax))[:, None, None, :]
    t = gs * np.asarray(qx).astype(F32) + np.asarray(qy).astype(F32) * F32(ay)
    if relu:
        t = np.maximum(t, F32(0))
    lo, hi = (0, 255) if out_dt == DT_UINT8 else (-128, 127)
    return np.clip(np.rint(t), lo, hi).astype(np.uint8 if out_dt == DT_UINT8 else np.int8)


# ------------------------------------------------------------------------------------------------ SE gate
def se_mean(x, dtype, scale=1.0):
    """Per-channel mean over h*w of x [n, h, w, C]. 8-bit: S = exact integer sum; ((float)S * scale [* 127/255 for u8])
    / hw in fp32 steps. Float kinds: float64 sum / hw (the walker's value; se_mean_ordered restates the device's fp32
    summation order)."""
    n, h, w, c = x.shape
    hw = F32(h * w)
    if dtype in (DT_INT8, DT_UINT8):
        s = np.asarray(x).astype(np.int64).sum(axis=(1, 2)).astype(F32) * F32(scale)
        if dtype == DT_UINT8:
            s = s * F32(127.0 / 255.0)
        return (s / hw).astype(F32)
    return (np.asarray(x, np.float64).sum(axis=(1, 2)).astype(F32) / hw).astype(F32)


_GATE_CLUSTER, _GATE_THREADS = 8, 256    # se.cu: CTAs per cluster, threads per CTA


def se_slots(ld, dtype_bytes):
    """Pooling slots of one gate CTA: the ld / L vectors of 16 bytes of a pixel spread over 256 threads."""
    nv = ld * dtype_bytes // 16
    return 1 if nv >= _GATE_THREADS else _GATE_THREADS // nv


def se_mean_ordered(x, ld):
    """The float gate's channel means in the device's order (se.cu, se_gate_kernel steps 1-2), float32 throughout:
    CTA `rank` of the 8-CTA cluster pools pixels [rank * chunk, min((rank + 1) * chunk, hw)), chunk = ceil(hw / 8);
    slot s of its `slots` (se_slots) sums every slots-th pixel from the first + s, starting from 0; the slot sums are
    added in slot order, then the 8 rank sums in rank order, then divided by hw. x [n, h, w, c] f32 or f16 (widened
    exactly); ld: stored channels of the tensor (only the slot count depends on it)."""
    n, h, w, c = x.shape
    hw = h * w
    v = np.asarray(x).reshape(n, hw, c).astype(F32)
    slots = se_slots(ld, np.asarray(x).dtype.itemsize)
    chunk = -(-hw // _GATE_CLUSTER)
    total = None
    with np.errstate(over="ignore", invalid="ignore"):
        for rank in range(_GATE_CLUSTER):
            px0 = min(rank * chunk, hw)
            px1 = min(px0 + chunk, hw)
            part = None
            for s in range(slots):
                acc = np.zeros((n, c), F32)
                for px in range(px0 + s, px1, slots):
                    acc = (acc + v[:, px]).astype(F32)
                part = acc if part is None else (part + acc).astype(F32)
            total = part if total is None else (total + part).astype(F32)
        return (total / F32(hw)).astype(F32)


def se_mean_depth(hw, ld, dtype_bytes):
    """Additions a pixel passes through in se_mean_ordered: its slot's pixels, the slot sums, the rank sums."""
    slots = se_slots(ld, dtype_bytes)
    chunk = -(-hw // _GATE_CLUSTER)
    return -(-chunk // slots) + slots + _GATE_CLUSTER


def se_gate_float(x, ld, w1, b1, w2, b2):
    """The float gate restated: se_mean_ordered, then se_hidden / se_excite below (which restate the device's
    squeeze and excitation orders and its explicit sigmoid)."""
    return se_excite(se_hidden(se_mean_ordered(x, ld), np.asarray(w1, F32), b1), np.asarray(w2, F32), b2)


def se_hidden(m, w1, b1):
    """relu(b1 + W1 . m) with the device's order: lane l sums c = l, l+32, ... in order, then a butterfly xor 16..1."""
    n, c = m.shape
    r = w1.shape[0]
    cp = (c + 31) // 32 * 32
    mp = np.zeros((n, cp), F32); mp[:, :c] = m
    wp = np.zeros((r, cp), F32); wp[:, :c] = w1
    p = np.zeros((n, r, 32), F32)
    for i in range(cp // 32):
        p = p + wp[None, :, 32 * i:32 * i + 32] * mp[:, None, 32 * i:32 * i + 32]
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        p = p + p[..., lane ^ o]
    h = p[..., 0] + np.asarray(b1, F32)[None]
    return np.maximum(h, F32(0)).astype(F32)


def se_excite(hid, w2, b2):
    """sigmoid(b2 + W2 . h), the dot product summed k = 0 .. r-1 in order."""
    n, r = hid.shape
    s = np.zeros((n, w2.shape[0]), F32)
    for k in range(r):
        s = s + w2[None, :, k] * hid[:, k:k + 1]
    return sigmoid_f32(s + np.asarray(b2, F32)[None])


def se_gate(x, dtype, scale, w1, b1, w2, b2):
    """The fused gate: x [n, h, w, C] -> fp32 [n, C]. w1 [r, C], w2 [C, r]."""
    return se_excite(se_hidden(se_mean(x, dtype, scale), np.asarray(w1, F32), b1), np.asarray(w2, F32), b2)


def se_gate_f64(x, w1, b1, w2, b2):
    """The same gate in float64 with a library sigmoid: what se_gate approximates."""
    m = np.asarray(x, np.float64).mean(axis=(1, 2))
    h = np.maximum(m @ np.asarray(w1, np.float64).T + np.asarray(b1, np.float64), 0)
    z = h @ np.asarray(w2, np.float64).T + np.asarray(b2, np.float64)
    return 1.0 / (1.0 + np.exp(-z))


# ------------------------------------------------------------------------------------------------ walker
class _G:
    def __init__(self, kind, head):
        self.kind, self.head, self.nodes = kind, head, [head]
        self.relu, self.relu_alpha = False, 0.0
        self.bn = self.scale = None
        self.out_name = head["name"]
        self.inputs = list(head["ins"])
        self.se = None            # SE gate: (down conv, up conv) nodes


def plan(graph):
    """Groups in execution order: conv [+BN] [+Scale] [+ReLU], Axpy [+ReLU], the SE gate chain, and the single ops."""
    nodes = {n["name"]: n for n in graph["nodes"]}
    consumed, groups = set(), []

    def sole(n):
        return nodes[n["outs"][0]] if len(n["outs"]) == 1 else None

    def se_chain(n):
        if n["op"] != "Pooling" or n["attrs"].get("method") != "AVG" or not n["attrs"].get("global_pooling"):
            return None
        down = sole(n)
        relu = sole(down) if down is not None and down["op"] == "Convolution" else None
        up = sole(relu) if relu is not None and relu["op"] == "ReLU" else None
        act = sole(up) if up is not None and up["op"] == "Convolution" else None
        axpy = sole(act) if act is not None and act["op"] == "Activation" and act["attrs"].get("type") == "Sigmoid" else None
        if axpy is None or axpy["op"] != "Axpy" or axpy["ins"][0] != act["name"]:
            return None
        return down, relu, up, act

    for n in graph["nodes"]:
        if n["name"] in consumed:
            continue
        op = n["op"]
        chain = se_chain(n) if op == "Pooling" else None
        if chain is not None:
            g = _G("se", n)
            g.se = (chain[0], chain[2])
            g.nodes += list(chain)
            g.out_name = chain[3]["name"]
        elif op == "Convolution":
            g = _G("conv", n)
            cur, nxt = n, sole(n)
            if nxt is not None and nxt["op"] == "BatchNorm":
                g.bn = nxt; g.nodes.append(nxt); cur, nxt = nxt, sole(nxt)
            if nxt is not None and nxt["op"] == "Scale":
                g.scale = nxt; g.nodes.append(nxt); cur, nxt = nxt, sole(nxt)
            if nxt is not None and nxt["op"] == "ReLU":
                g.relu, g.relu_alpha = True, float(nxt["attrs"].get("alpha", 0.0)); g.nodes.append(nxt); cur = nxt
            g.out_name = cur["name"]
        elif op in ("Axpy", "Dense"):
            g = _G(op.lower(), n)
            nxt = sole(n)
            if nxt is not None and nxt["op"] == "ReLU":
                g.relu, g.relu_alpha = True, float(nxt["attrs"].get("alpha", 0.0))
                g.nodes.append(nxt); g.out_name = nxt["name"]
        else:
            kind = {"Pooling": "pool", "Softmax": "softmax", "Input": "input", "Output": "output", "Split": "split"}.get(op)
            if kind is None:
                raise NotImplementedError("SE walker: op %s" % op)
            g = _G(kind, n)
        for m in g.nodes:
            consumed.add(m["name"])
        groups.append(g)
    return groups


def _se_weights(g):
    down, up = g.se
    r, c = int(down["attrs"]["filter_num"]), int(up["attrs"]["filter_num"])
    w1 = W._attr_tensor(down["attrs"]["weight_1"]).reshape(r, c)
    b1 = W._attr_tensor(down["attrs"]["weight_2"]).reshape(-1)
    w2 = W._attr_tensor(up["attrs"]["weight_1"]).reshape(c, r)
    b2 = W._attr_tensor(up["attrs"]["weight_2"]).reshape(-1)
    return w1, b1, w2, b2


def _pool_args(a):
    return ((tuple(a["pool_size"]), tuple(a["padding"]), tuple(a["strides"]), {"MAX": 1, "AVG": 2, "AVGEXC": 3}[a["method"]]),
            dict(global_pooling=bool(a["global_pooling"]), floor_as_conv=bool(a.get("cmp_out_shape_floor_as_conv", False))))


def _dense_in(x):
    if x.ndim == 4:
        x = np.transpose(x, (0, 3, 1, 2))       # Dense flattens in NCHW order (saber_fc.cu:27-35)
    return np.ascontiguousarray(x).reshape(x.shape[0], -1)


def _output(v):
    return v.reshape(v.shape[0], -1) if v.shape[1] == 1 and v.shape[2] == 1 else np.transpose(v, (0, 3, 1, 2))


def run_fp32(graph, x_nchw, return_values=False, collect_absmax=False, fast=False):
    """FP32 forward (NHWC inside). Returns {output: array}; with return_values also {node: value}; with
    collect_absmax also {node: max|x|} (the max-abs calibration of oracle/model_walker.py)."""
    vals, absmax, outputs = {}, {}, {}

    def put(g, v):
        for m in g.nodes:
            vals[m["name"]] = v
            if collect_absmax:
                absmax[m["name"]] = float(np.abs(v).max())

    for g in plan(graph):
        a = g.head["attrs"]
        if g.kind == "input":
            put(g, np.ascontiguousarray(np.transpose(np.asarray(x_nchw, F32), (0, 2, 3, 1))))
        elif g.kind == "split":
            put(g, vals[g.inputs[0]])
        elif g.kind == "conv":
            w, bias = W._folded_conv_weights(g)
            put(g, O.conv_f32_nhwc(vals[g.inputs[0]], w, bias, group=int(a["group"]), relu=g.relu,
                                   neg_slope=g.relu_alpha, fast=fast, **W._conv_kw(a)))
        elif g.kind == "se":
            x = vals[g.inputs[0]]
            gate = se_gate(x, DT_FLOAT, 1.0, *_se_weights(g))
            put(g, gate.reshape(gate.shape[0], 1, 1, -1))
        elif g.kind == "axpy":
            gate = vals[g.inputs[0]].reshape(vals[g.inputs[0]].shape[0], -1)
            put(g, axpy_f32(gate, vals[g.inputs[1]], vals[g.inputs[2]], g.relu, g.relu_alpha))
        elif g.kind == "pool":
            args, kw = _pool_args(a)
            put(g, O.pool_f32(vals[g.inputs[0]], *args, nhwc=True, **kw))
        elif g.kind == "dense":
            w = W._attr_tensor(a["weight_1"]).reshape(int(a["out_dim"]), -1)
            b = W._attr_tensor(a["weight_2"]).reshape(-1) if a.get("bias_term") else None
            y = O.fc_f32(_dense_in(vals[g.inputs[0]]), w, b)
            if g.relu:
                y = O.activation_f32(y, 2, g.relu_alpha)
            put(g, y.reshape(y.shape[0], 1, 1, -1))
        elif g.kind == "softmax":
            x = vals[g.inputs[0]]
            n = x.shape[0]
            put(g, O.softmax_f32(x.reshape(n, -1), n, x.size // n, 1).reshape(x.shape))
        elif g.kind == "output":
            outputs[g.head["name"]] = _output(vals[g.inputs[0]])
    if return_values:
        return outputs, vals
    if collect_absmax:
        return outputs, absmax
    return outputs


def calibrate(graph, images_nchw, fast=False):
    """Max-abs calibration: scale = max|x| / 127 per node output."""
    _, absmax = run_fp32(graph, images_nchw, collect_absmax=True, fast=fast)
    return {k: (v / 127.0 if v > 0 else 1.0) for k, v in absmax.items()}


def run_int8(graph, x_nchw, edge_scales, return_intermediate=False, fast=False):
    """INT8 forward, x86 Saber semantics as oracle/model_walker.run_int8, with the fp32 SE gate and the INT8 Axpy rule.
    trace: {group head and last node: (array NHWC, dtype code, scale)}."""
    from anakin_b200 import modelzoo
    nodes = {n["name"]: n for n in graph["nodes"]}
    vals, outputs, trace = {}, {}, {}
    gates = modelzoo._se_gate_sigmoids(graph)

    def node_is_int8(name):
        # an unmarked graph: the INT8 marking of modelzoo.apply_int8
        bt = nodes[name].get("bit_type")
        return bt == "INT8" if bt is not None else (nodes[name]["op"] in modelzoo.INT8_OPS or name in gates)

    def put(g, arr, dt, scale):
        for m in g.nodes:
            vals[m["name"]] = (arr, dt, scale)
        trace[g.out_name] = trace[g.head["name"]] = (arr, dt, scale)

    def as_float(v):
        arr, dt, sc = v
        if dt == DT_FLOAT:
            return arr
        f = arr.astype(F32) * F32(sc)
        return f * F32(127.0 / 255.0) if dt == DT_UINT8 else f

    for g in plan(graph):
        a = g.head["attrs"]
        if g.kind == "input":
            put(g, np.ascontiguousarray(np.transpose(np.asarray(x_nchw, F32), (0, 2, 3, 1))), DT_FLOAT,
                edge_scales[g.out_name])
        elif g.kind == "split":
            put(g, *vals[g.inputs[0]])
        elif g.kind in ("conv", "dense"):
            src, sdt, s_in = vals[g.inputs[0]]
            if g.kind == "conv":
                w, bias = W._folded_conv_weights(g)
                kw = W._conv_kw(a)
                kw["group"] = int(a["group"])
            else:
                w = W._attr_tensor(a["weight_1"]).reshape(int(a["out_dim"]), -1)
                if src.ndim == 4 and src.shape[1] * src.shape[2] > 1:
                    n_, h_, w_, c_ = src.shape
                    w = w.reshape(-1, c_, h_, w_).transpose(0, 2, 3, 1).reshape(w.shape[0], -1)
                    src = src.reshape(n_, 1, 1, -1)
                w = w.reshape(w.shape[0], -1, 1, 1)
                bias = W._attr_tensor(a["weight_2"]).reshape(-1) if a.get("bias_term") else np.zeros(w.shape[0], F32)
                kw = dict(stride=(1, 1), pad=(0, 0), dil=(1, 1))
            if sdt == DT_FLOAT:
                src, sdt = O.quant_fp32_s8(src, s_in), DT_INT8
            wq, w_scale = O.quant_weights_per_oc(w)
            s_out = edge_scales[g.out_name]
            outs = nodes[g.out_name]["outs"]
            int8_out = len(outs) > 0 and all(node_is_int8(o) for o in outs)
            out_dt = (DT_UINT8 if g.relu else DT_INT8) if int8_out else DT_FLOAT
            scale, bias_f, sum_scale = O.int8_conv_scales(w_scale, bias, s_in, sdt, s_out, out_dt, 1.0, DT_INT8)
            y = O.conv_s8_nhwc_x86(src, wq, bias_f, scale, residual=None, sum_scale=sum_scale, out_dtype=out_dt,
                                   relu=g.relu, fast=fast, **kw)
            put(g, y, out_dt, s_out)
        elif g.kind == "se":
            x, dt, sc = vals[g.inputs[0]]
            gate = se_gate(x, dt, sc, *_se_weights(g))
            put(g, gate.reshape(gate.shape[0], 1, 1, -1), DT_FLOAT, 1.0)
        elif g.kind == "axpy":
            gate = vals[g.inputs[0]][0].reshape(vals[g.inputs[0]][0].shape[0], -1)
            (qx, dx, sx), (qy, dy, sy) = vals[g.inputs[1]], vals[g.inputs[2]]
            s_out = edge_scales[g.out_name]
            out_dt = DT_UINT8 if g.relu else DT_INT8
            ax, ay = axpy_factors(sx, dx, sy, dy, s_out, out_dt)
            put(g, axpy_q8(gate, qx, qy, ax, ay, out_dt, g.relu), out_dt, s_out)
        elif g.kind == "pool":
            src, sdt, s_in = vals[g.inputs[0]]
            args, kw = _pool_args(a)
            if sdt == DT_FLOAT:
                put(g, O.pool_f32(src, *args, nhwc=True, **kw), DT_FLOAT, s_in)
            else:
                put(g, O.pool_s8_nhwc(src, *args, fast=fast, **kw), sdt, s_in)
        elif g.kind == "softmax":
            x = as_float(vals[g.inputs[0]])
            n = x.shape[0]
            put(g, O.softmax_f32(x.reshape(n, -1), n, x.size // n, 1).reshape(x.shape), DT_FLOAT, 1.0)
        elif g.kind == "output":
            outputs[g.head["name"]] = _output(as_float(vals[g.inputs[0]]))
    if return_intermediate:
        return outputs, trace
    return outputs
