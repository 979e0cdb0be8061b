"""Synthetic benchmark models in Anakin's own graph format.

The reference ships no model files (SURVEY.md section 0), so the benchmark networks are
synthesised here exactly as the reference's converter (tools/external_converter_v2) would
emit them from the Caffe prototxts: op names and attribute names per
tools/external_converter_v2/parser/operations/ops.py:9-181, weights as `weight_N` TENSOR
attributes (framework/operators/convolution.cpp:32-66, batch_norm.cpp:36-39, scale.cpp:41-47,
dense.cpp:20-33), explicit `Split` nodes on fan-out, Caffe-style ResNet (stride on the
first 1x1 of a stage, 3x3/s2 ceil-mode max pool).  Weights are He-normal, seed 1234
(SURVEY.md section 8d) -- deterministic, so every rank / the oracle / the GPU box build
bit-identical models.
"""
import json
import os

import numpy as np

from . import anakin_bin


class GraphBuilder:
    def __init__(self, name, seed=1234):
        self.name = name
        self.rng = np.random.default_rng(seed)
        self.nodes = []      # (name, op, [input node names], attrs)
        self.index = {}

    def add(self, name, op, ins, **attrs):
        assert name not in self.index, name
        self.index[name] = len(self.nodes)
        self.nodes.append({"name": name, "op": op, "ins": list(ins), "outs": [], "attrs": dict(attrs),
                           "bit_type": None, "lane": 0, "need_wait": False})
        return name

    # ---- layer helpers (attr schema = ops.py)
    def input(self, name, shape):
        return self.add(name, "Input", [], input_shape=[int(s) for s in shape], max_len=0, max_batch=0,
                        alias="NULL", data_type="NULL", layout="NCHW")

    def conv(self, name, bottom, cin, cout, k, stride=1, pad=0, bias=False, group=1, dilation=1):
        fan_in = (cin // group) * k * k
        w = (self.rng.standard_normal((cout, cin // group, k, k)) * np.sqrt(2.0 / fan_in)).astype(np.float32)
        attrs = dict(filter_num=int(cout), kernel_size=[k, k], strides=[stride, stride], padding=[pad, pad],
                     dilation_rate=[dilation, dilation], group=int(group), axis=1, bias_term=bool(bias),
                     weight_1=w)
        if bias:
            attrs["weight_2"] = self.rng.uniform(-0.1, 0.1, (1, cout, 1, 1)).astype(np.float32)
        return self.add(name, "Convolution", [bottom], **attrs)

    def batchnorm(self, name, bottom, c):
        mean = self.rng.uniform(-0.1, 0.1, (1, c, 1, 1)).astype(np.float32)
        var = self.rng.uniform(0.5, 1.5, (1, c, 1, 1)).astype(np.float32)
        factor = np.ones((1, 1, 1, 1), np.float32)
        return self.add(name, "BatchNorm", [bottom], momentum=0.999, epsilon=1e-5, weight_1=mean,
                        weight_2=var, weight_3=factor)

    def scale(self, name, bottom, c, gamma_range=(0.8, 1.2)):
        gamma = self.rng.uniform(gamma_range[0], gamma_range[1], (1, c, 1, 1)).astype(np.float32)
        beta = self.rng.uniform(-0.1, 0.1, (1, c, 1, 1)).astype(np.float32)
        return self.add(name, "Scale", [bottom], axis=1, num_axes=1, bias_term=True, weight_1=gamma,
                        weight_2=beta)

    def relu(self, name, bottom, alpha=0.0):
        return self.add(name, "ReLU", [bottom], alpha=float(alpha))

    def pool(self, name, bottom, k, stride, pad=0, method="MAX", global_pooling=False):
        return self.add(name, "Pooling", [bottom], pool_size=[k, k], strides=[stride, stride],
                        padding=[pad, pad], method=method, global_pooling=bool(global_pooling),
                        cmp_out_shape_floor_as_conv=False)

    def eltwise_add(self, name, a, b):
        return self.add(name, "Eltwise", [a, b], type="Add", coeff=[1.0, 1.0])

    def dense(self, name, bottom, cin, cout, gain=1.0):
        w = (self.rng.standard_normal((1, 1, cout, cin)) * (gain * np.sqrt(1.0 / cin))).astype(np.float32)
        b = self.rng.uniform(-0.1, 0.1, (1, cout, 1, 1)).astype(np.float32)
        return self.add(name, "Dense", [bottom], out_dim=int(cout), axis=1, bias_term=True, weight_1=w,
                        weight_2=b)

    def softmax(self, name, bottom):
        return self.add(name, "Softmax", [bottom], axis=1)

    def sigmoid(self, name, bottom):
        return self.add(name, "Activation", [bottom], type="Sigmoid")

    def axpy(self, name, gate, x, y):
        """Caffe SENet's Axpy layer (converter: caffe_layer_param_transmit.py): out = gate[n,c] * x + y."""
        return self.add(name, "Axpy", [gate, x, y])

    def se_gate(self, prefix, bottom, c, reduction=16):
        """Squeeze-and-excitation gate: global AVE pooling, 1x1 conv C -> C/r with bias, ReLU, 1x1 conv C/r -> C with
        bias, Sigmoid."""
        x = self.pool(prefix + "_pool", bottom, 1, 1, 0, "AVG", global_pooling=True)
        x = self.conv(prefix + "_down", x, c, c // reduction, 1, bias=True)
        x = self.relu(prefix + "_down_relu", x)
        x = self.conv(prefix + "_up", x, c // reduction, c, 1, bias=True)
        return self.sigmoid(prefix + "_prob", x)

    def output(self, name, bottom):
        return self.add(name, "Output", [bottom])

    def conv_bn_scale(self, prefix, bottom, cin, cout, k, stride, pad, relu, bias=False, group=1,
                      gamma_range=(0.8, 1.2)):
        x = self.conv(prefix, bottom, cin, cout, k, stride, pad, bias=bias, group=group)
        x = self.batchnorm("bn_" + prefix, x, cout)
        x = self.scale("scale_" + prefix, x, cout, gamma_range)
        if relu:
            x = self.relu(prefix + "_relu", x)
        return x

    # ---- finalize: insert Split nodes on fan-out (as the converter does), wire ins/outs/edges
    def finalize(self):
        consumers = {}
        for n in self.nodes:
            for b in n["ins"]:
                consumers.setdefault(b, []).append(n["name"])
        nodes = []
        rename = {}  # (producer, consumer) -> actual bottom name
        for n in self.nodes:
            nodes.append(n)
            cons = consumers.get(n["name"], [])
            if len(cons) > 1:
                sp = {"name": n["name"] + "_split", "op": "Split", "ins": [n["name"]], "outs": [],
                      "attrs": {"split_num": len(cons)}, "bit_type": None, "lane": 0, "need_wait": False}
                nodes.append(sp)
                for c in cons:
                    rename[(n["name"], c)] = sp["name"]
        for n in nodes:
            if n["op"] != "Split":
                n["ins"] = [rename.get((b, n["name"]), b) for b in n["ins"]]
        byname = {n["name"]: n for n in nodes}
        for n in nodes:
            n["outs"] = []
        for n in nodes:
            for b in n["ins"]:
                byname[b]["outs"].append(n["name"])
        g = {"name": self.name, "nodes": nodes,
             "ins": [n["name"] for n in nodes if n["op"] == "Input"],
             "outs": [n["name"] for n in nodes if n["op"] == "Output"],
             "edges_in": {n["name"]: [(b, None) for b in n["ins"]] for n in nodes if n["ins"]},
             "edges_out": {n["name"]: [(t, None) for t in n["outs"]] for n in nodes if n["outs"]},
             "edges_info": {}, "version": (2, 0, 0, 200), "is_optimized": False}
        return g


# --------------------------------------------------------------------------- networks
def resnet(depth=50, batch=1, seed=1234, num_classes=1000):
    blocks = {50: [3, 4, 6, 3], 101: [3, 4, 23, 3]}[depth]
    g = GraphBuilder("ResNet-%d" % depth, seed)
    x = g.input("input_0", (batch, 3, 224, 224))
    x = g.conv_bn_scale("conv1", x, 3, 64, 7, 2, 3, relu=True, bias=True)
    x = g.pool("pool1", x, 3, 2, 0, "MAX")
    cin = 64
    for si, nblk in enumerate(blocks):
        mid = 64 << si
        cout = mid * 4
        for bi in range(nblk):
            if depth == 50 or nblk <= 6:
                tag = "%d%s" % (si + 2, "abcdefgh"[bi])
            else:
                tag = "%d%s" % (si + 2, "a" if bi == 0 else "b%d" % bi)
            stride = 2 if (bi == 0 and si > 0) else 1
            if bi == 0:
                short = g.conv_bn_scale("res%s_branch1" % tag, x, cin, cout, 1, stride, 0, relu=False,
                                        gamma_range=(0.5, 0.7))
            else:
                short = x
            y = g.conv_bn_scale("res%s_branch2a" % tag, x, cin, mid, 1, stride, 0, relu=True)
            y = g.conv_bn_scale("res%s_branch2b" % tag, y, mid, mid, 3, 1, 1, relu=True)
            # small gamma on the residual-branch tail (and a damped projection shortcut) keeps the
            # randomly initialised net's activations O(1) through 16/33 residual sums
            y = g.conv_bn_scale("res%s_branch2c" % tag, y, mid, cout, 1, 1, 0, relu=False,
                                gamma_range=(0.15, 0.3))
            x = g.eltwise_add("res%s" % tag, short, y)
            x = g.relu("res%s_relu" % tag, x)
            cin = cout
    x = g.pool("pool5", x, 7, 1, 0, "AVG", global_pooling=True)
    x = g.dense("fc1000", x, cin, num_classes, gain=6.0)
    x = g.softmax("prob", x)
    g.output("prob_out", x)
    return g.finalize()


def _se_bottleneck(g, tag, x, cin, mid, stride, project, gamma_range=(0.15, 0.3), short_gamma=(0.5, 0.7)):
    """One SE-ResNet bottleneck: the ResNet block with the SE gate scaling branch2c before the residual sum
    (out = ReLU(Axpy(gate, branch2c, shortcut)))."""
    cout = mid * 4
    short = g.conv_bn_scale("res%s_branch1" % tag, x, cin, cout, 1, stride, 0, relu=False,
                            gamma_range=short_gamma) if project else x
    y = g.conv_bn_scale("res%s_branch2a" % tag, x, cin, mid, 1, stride, 0, relu=True)
    y = g.conv_bn_scale("res%s_branch2b" % tag, y, mid, mid, 3, 1, 1, relu=True)
    y = g.conv_bn_scale("res%s_branch2c" % tag, y, mid, cout, 1, 1, 0, relu=False, gamma_range=gamma_range)
    gate = g.se_gate("res%s_se" % tag, y, cout)
    x = g.axpy("res%s" % tag, gate, y, short)
    return g.relu("res%s_relu" % tag, x)


def se_resnet(depth=50, batch=1, seed=1234, num_classes=1000):
    """SE-ResNet (Hu et al., "Squeeze-and-Excitation Networks"): resnet(depth)'s Caffe topology with an SE gate of
    reduction 16 on every bottleneck, written with the Axpy layer as the Caffe SENet models are."""
    blocks = {50: [3, 4, 6, 3]}[depth]
    g = GraphBuilder("SE-ResNet-%d" % depth, seed)
    x = g.input("input_0", (batch, 3, 224, 224))
    x = g.conv_bn_scale("conv1", x, 3, 64, 7, 2, 3, relu=True, bias=True)
    x = g.pool("pool1", x, 3, 2, 0, "MAX")
    cin = 64
    for si, nblk in enumerate(blocks):
        mid = 64 << si
        for bi in range(nblk):
            tag = "%d%s" % (si + 2, "abcdefgh"[bi])
            x = _se_bottleneck(g, tag, x, cin, mid, 2 if (bi == 0 and si > 0) else 1, bi == 0)
            cin = mid * 4
    x = g.pool("pool5", x, 7, 1, 0, "AVG", global_pooling=True)
    x = g.dense("fc1000", x, cin, num_classes, gain=6.0)
    x = g.softmax("prob", x)
    g.output("prob_out", x)
    return g.finalize()


def tiny_se_resnet(batch=1, seed=13, hw=32, num_classes=10):
    """tiny_resnet with an SE gate on every block: every op kind of SE-ResNet-50 (stem conv+pool, projection shortcut,
    stride-2 stage, SE gate, Axpy, global pool, fc, softmax) at a size the CPU oracle walks in milliseconds."""
    g = GraphBuilder("TinySEResNet", seed)
    x = g.input("input_0", (batch, 3, hw, hw))
    x = g.conv_bn_scale("conv1", x, 3, 16, 7, 2, 3, relu=True, bias=True)
    x = g.pool("pool1", x, 3, 2, 0, "MAX")
    cin = 16
    for si, nblk in enumerate([2, 2]):
        mid = 16 << si
        for bi in range(nblk):
            tag = "%d%s" % (si + 2, "ab"[bi])
            x = _se_bottleneck(g, tag, x, cin, mid, 2 if (bi == 0 and si > 0) else 1, bi == 0, short_gamma=(0.8, 1.2))
            cin = mid * 4
    x = g.pool("pool5", x, 7, 1, 0, "AVG", global_pooling=True)
    x = g.dense("fc", x, cin, num_classes, gain=3.0)
    x = g.softmax("prob", x)
    g.output("prob_out", x)
    return g.finalize()


def vgg16(batch=1, seed=1234, num_classes=1000):
    g = GraphBuilder("VGG16", seed)
    x = g.input("input_0", (batch, 3, 224, 224))
    cfg = [(2, 64), (2, 128), (3, 256), (3, 512), (3, 512)]
    cin = 3
    for si, (n, c) in enumerate(cfg):
        for ci in range(n):
            name = "conv%d_%d" % (si + 1, ci + 1)
            x = g.conv(name, x, cin, c, 3, 1, 1, bias=True)
            x = g.relu("relu%d_%d" % (si + 1, ci + 1), x)
            cin = c
        x = g.pool("pool%d" % (si + 1), x, 2, 2, 0, "MAX")
    x = g.dense("fc6", x, 512 * 7 * 7, 4096)
    x = g.relu("relu6", x)
    x = g.dense("fc7", x, 4096, 4096)
    x = g.relu("relu7", x)
    x = g.dense("fc8", x, 4096, num_classes)
    x = g.softmax("prob", x)
    g.output("prob_out", x)
    return g.finalize()


def mobilenet_v1(batch=1, seed=1234, num_classes=1000):
    g = GraphBuilder("MobileNet-v1", seed)
    x = g.input("input_0", (batch, 3, 224, 224))
    x = g.conv_bn_scale("conv1", x, 3, 32, 3, 2, 1, relu=True)
    cfg = [(32, 64, 1), (64, 128, 2), (128, 128, 1), (128, 256, 2), (256, 256, 1), (256, 512, 2)] + \
          [(512, 512, 1)] * 5 + [(512, 1024, 2), (1024, 1024, 1)]
    for i, (cin, cout, s) in enumerate(cfg):
        x = g.conv_bn_scale("conv%d_dw" % (i + 2), x, cin, cin, 3, s, 1, relu=True, group=cin)
        x = g.conv_bn_scale("conv%d_sep" % (i + 2), x, cin, cout, 1, 1, 0, relu=True)
    x = g.pool("pool6", x, 7, 1, 0, "AVG", global_pooling=True)
    x = g.dense("fc7", x, 1024, num_classes)
    x = g.softmax("prob", x)
    g.output("prob_out", x)
    return g.finalize()


def tiny_resnet(batch=1, seed=7, hw=32, num_classes=10):
    """A 2-stage bottleneck net with every op kind of ResNet-50 (stem conv+pool, projection
    shortcut, stride-2 stage, global pool, fc, softmax); small enough for the CPU oracle
    in milliseconds -- used by smoke() and the fast parity tests."""
    g = GraphBuilder("TinyResNet", seed)
    x = g.input("input_0", (batch, 3, hw, hw))
    x = g.conv_bn_scale("conv1", x, 3, 16, 7, 2, 3, relu=True, bias=True)
    x = g.pool("pool1", x, 3, 2, 0, "MAX")
    cin = 16
    for si, nblk in enumerate([2, 2]):
        mid = 16 << si
        cout = mid * 4
        for bi in range(nblk):
            tag = "%d%s" % (si + 2, "ab"[bi])
            stride = 2 if (bi == 0 and si > 0) else 1
            short = g.conv_bn_scale("res%s_branch1" % tag, x, cin, cout, 1, stride, 0, relu=False) if bi == 0 else x
            y = g.conv_bn_scale("res%s_branch2a" % tag, x, cin, mid, 1, stride, 0, relu=True)
            y = g.conv_bn_scale("res%s_branch2b" % tag, y, mid, mid, 3, 1, 1, relu=True)
            y = g.conv_bn_scale("res%s_branch2c" % tag, y, mid, cout, 1, 1, 0, relu=False,
                                gamma_range=(0.15, 0.3))
            x = g.eltwise_add("res%s" % tag, short, y)
            x = g.relu("res%s_relu" % tag, x)
            cin = cout
    x = g.pool("pool5", x, 7, 1, 0, "AVG", global_pooling=True)
    x = g.dense("fc", x, cin, num_classes, gain=3.0)
    x = g.softmax("prob", x)
    g.output("prob_out", x)
    return g.finalize()


def tiny_mobilenet(batch=1, seed=11, hw=32, num_classes=10):
    """MobileNet-v1 in miniature: 3x3/s2 stem, four depthwise-separable pairs (stride 1 and 2, 32..256 channels), global
    average pool, fc, softmax -- every op kind of MobileNet-v1 at a size the CPU oracle walks in milliseconds (the INT8
    depthwise path of the net is checked on it)."""
    g = GraphBuilder("TinyMobileNet", seed)
    x = g.input("input_0", (batch, 3, hw, hw))
    x = g.conv_bn_scale("conv1", x, 3, 32, 3, 2, 1, relu=True)
    cfg = [(32, 64, 1), (64, 128, 2), (128, 128, 1), (128, 256, 2)]
    for i, (cin, cout, s) in enumerate(cfg):
        x = g.conv_bn_scale("conv%d_dw" % (i + 2), x, cin, cin, 3, s, 1, relu=True, group=cin)
        x = g.conv_bn_scale("conv%d_sep" % (i + 2), x, cin, cout, 1, 1, 0, relu=True)
    x = g.pool("pool6", x, hw // 8, 1, 0, "AVG", global_pooling=True)
    x = g.dense("fc7", x, 256, num_classes, gain=3.0)
    x = g.softmax("prob", x)
    g.output("prob_out", x)
    return g.finalize()


BUILDERS = {
    "resnet50": lambda batch=1, seed=1234: resnet(50, batch, seed),
    "resnet101": lambda batch=1, seed=1234: resnet(101, batch, seed),
    "vgg16": vgg16,
    "mobilenet_v1": mobilenet_v1,
    "tiny_resnet": lambda batch=1, seed=7: tiny_resnet(batch, seed),
    "tiny_mobilenet": lambda batch=1, seed=11: tiny_mobilenet(batch, seed),
    "se_resnet50": lambda batch=1, seed=1234: se_resnet(50, batch, seed),
    "tiny_se_resnet": lambda batch=1, seed=13: tiny_se_resnet(batch, seed),
}


def synthetic_input(batch, hw=224, seed=42):
    """fp32 NCHW in [-1,1], image i seeded 42+i (SURVEY.md section 8d; value range of the
    reference example, examples/cuda/example_nv_cnn_net.cpp:48).  Each image is a per-channel
    offset + a coarse 7x7 pattern + uniform noise, so that different images give different
    logits (pure i.i.d. noise averages out in the global pool and every image ties)."""
    out = np.empty((batch, 3, hw, hw), np.float32)
    for i in range(batch):
        rng = np.random.default_rng(seed + i)
        base = rng.uniform(-0.45, 0.45, (3, 1, 1))
        coarse = rng.uniform(-0.3, 0.3, (3, 7, 7))
        rep = (hw + 6) // 7
        coarse = np.repeat(np.repeat(coarse, rep, axis=1), rep, axis=2)[:, :hw, :hw]
        noise = rng.uniform(-0.25, 0.25, (3, hw, hw))
        out[i] = (base + coarse + noise).astype(np.float32)
    return out


# --------------------------------------------------------------------------- INT8 annotation
INT8_OPS = {"Convolution", "BatchNorm", "Scale", "ReLU", "Pooling", "Eltwise", "Dense", "Split", "Input", "Axpy"}


def _se_gate_sigmoids(graph):
    """Sigmoid Activation nodes read as the gate (input 0) of an Axpy: the tail of an SE gate chain."""
    by = {n["name"]: n for n in graph["nodes"]}
    return {n["ins"][0] for n in graph["nodes"]
            if n["op"] == "Axpy" and n["ins"] and by[n["ins"][0]]["op"] == "Activation"}


def apply_int8(graph, edge_scales):
    """Mark nodes INT8 (NodeProto.bit_type, node.proto:44) and write the calibrated edge scales
    (TargetProto.scale, graph.proto:52-56) -- what the converter does with a calibration table.
    edge_scales: {producer_node_name: scale} where scale = max|x|/127 of that node's output.
    The Sigmoid of an SE gate is marked too, so that the whole gate chain -- fused into one SqueezeExcite node, which
    reads the 8-bit block output -- is INT8 (its output is an fp32 gate all the same)."""
    gates = _se_gate_sigmoids(graph)
    for n in graph["nodes"]:
        n["bit_type"] = "INT8" if n["op"] in INT8_OPS or n["name"] in gates else "FLOAT"
    for key in ("edges_in", "edges_out"):
        for name, targets in graph[key].items():
            new = []
            for other, _ in targets:
                producer = other if key == "edges_in" else name
                sc = edge_scales.get(producer)
                new.append((other, [float(sc)] if sc is not None else None))
            graph[key][name] = new
    return graph


_GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def load_calibration(model_name):
    """Frozen max-abs calibration table (tests/golden/<model>_calib.json, produced by
    tools/make_golden.py from the fp32 CPU oracle over 8 synthetic images)."""
    p = os.path.join(_GOLDEN, "%s_calib.json" % model_name)
    with open(p) as f:
        return json.load(f)["edge_scales"]


HEAD_DENSE = {"tiny_resnet": "fc", "resnet50": "fc1000", "resnet101": "fc1000", "vgg16": "fc8", "mobilenet_v1": "fc7",
              "tiny_mobilenet": "fc7", "se_resnet50": "fc1000", "tiny_se_resnet": "fc"}


def center_head(graph, model_name):
    """A randomly initialised net maps every image to nearly the same logits (the classifier sees a large common
    feature vector plus a small image-dependent part), so top-1 would be the same class for every input and an
    "exact top-1" check would discriminate nothing. The classifier bias is therefore chosen as b - W.mu, mu = the mean
    penultimate feature vector of the 8 calibration images (tools/make_golden.py computes it with the fp32 oracle and
    commits it as tests/golden/<model>_fc_bias.npy): logits are centred and the arg-max varies from image to image.
    Architecture and every other weight are untouched."""
    p = os.path.join(_GOLDEN, "%s_fc_bias.npy" % model_name)
    if not os.path.exists(p):
        return graph
    bias = np.load(p).astype(np.float32)
    for n in graph["nodes"]:
        if n["name"] == HEAD_DENSE[model_name]:
            assert n["attrs"]["weight_2"].size == bias.size
            n["attrs"]["weight_2"] = bias.reshape(n["attrs"]["weight_2"].shape)
    return graph


def build(model_name, batch=1, precision="fp32", centered=True):
    g = BUILDERS[model_name](batch)
    if centered:
        center_head(g, model_name)
    if precision == "int8":
        apply_int8(g, load_calibration(model_name))
    return g


def save(graph, path):
    anakin_bin.save(graph, path)
