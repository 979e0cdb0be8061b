"""Every edge of the FP32 and FP16 nets, bit for bit, on designed weights whose sums are exact (net_exact.py).

On such data the kernels' results do not depend on accumulation order, plan, tile width or split-K, so the exact walk
predicts each edge; the comparison has no tolerance. What it covers sits above the kernels: the BatchNorm / Scale fold
and its cache shared by the FP32 and FP16 Nets of one Graph, biases and residuals, the Dense flatten order, pooling
divisors, padded channels, the fp16 edge dtypes and the order of the images of a batch.

ResNet-50 / 101 and MobileNet-v1 run at 256 x 256 (Graph.Reshape): their 8 x 8 global average divides exactly, where
224 x 224's 7 x 7 window would leave full-mantissa values in front of the classifier (see net_exact.NETS).
"""
import numpy as np
import pytest

import net_exact as E

pytestmark = pytest.mark.gpu

CASES = [(n, b) for n in ("tiny_resnet", "tiny_mobilenet") for b in (1, 3, 8)] + \
    [("resnet50", 1), ("resnet50", 3), ("resnet101", 1), ("vgg16", 1), ("mobilenet_v1", 1)]
DT = {0: np.float16, 1: np.float32}      # tensor_info dtype codes


def _graph(graph, name, batch):
    from anakin_b200 import anakin_bin, api
    G = api.Graph.from_bytes(anakin_bin.dumps(graph))
    G.ResetBatchSize("input_0", batch)
    hw = E.NETS[name]
    G.Reshape("input_0", [batch, 3, hw, hw])
    G.Optimize()
    return G


def _run(net, x, times=1):
    net.set_input("input_0", x)
    for _ in range(times):
        net.prediction()
    net.sync()


def _bits(a):
    """Bits of a float array with -0 read as +0: the kernels' zero signs are checked bit for bit by the kernel tests;
    here a ReLU's -0 and a pooling's choice among zeros would only obscure the comparison."""
    a = np.where(a == 0, np.zeros((), a.dtype), a).astype(a.dtype)
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


def _pooled_by(graph, conv):
    """The Pooling node a fused conv + pooling op (op name ending in "Pool") holds the output of."""
    nodes = {n["name"]: n for n in graph["nodes"]}
    n = nodes[conv]
    while n["op"] != "Pooling":
        assert len(n["outs"]) == 1, conv
        n = nodes[n["outs"][0]]
    return n["name"]


def _valid(arr, info, shape):
    """The valid channels of a read tensor in the walk's shape (NHWC, or [n, 1, 1, k])."""
    n, c, h, w = info["dims"]
    if info["layout"] == 9:
        return arr[..., :c].reshape(shape)
    return np.ascontiguousarray(np.transpose(arr, (0, 2, 3, 1))).reshape(shape)


def _check_edges(net, graph, wk, what):
    """Every launched op's edge against the walk: valid channels bit for bit, padded channels zero. Returns (edges,
    elements) compared."""
    edges = elems = 0
    for name, op in net.exec_order():
        if op == "Softmax":
            continue
        node = _pooled_by(graph, name) if op.endswith("Pool") else name
        assert node in wk.vals, "%s: %s (%s) has no value in the walk" % (what, name, op)
        want = wk.vals[node]
        arr, info = net.read_tensor(name)
        assert DT.get(info["dtype"]) == want.dtype, (what, name, op, info["dtype"], want.dtype)
        got = _valid(arr, info, want.shape)
        if info["layout"] == 9:
            assert (arr[..., info["dims"][1]:] == 0).all(), "%s: %s writes its padded channels" % (what, name)
        bad = np.argwhere(_bits(got) != _bits(want))
        assert bad.shape[0] == 0, "%s: %s (%s): %d of %d values differ, first at %s: %r, want %r" % (
            what, name, op, bad.shape[0], want.size, bad[0], got[tuple(bad[0])], want[tuple(bad[0])])
        edges += 1
        elems += want.size
    return edges, elems


@pytest.mark.parametrize("name,batch", CASES)
def test_net_edges_exact(name, batch):
    from anakin_b200 import api
    from float_ops_ref import rows_adds, softmax_bound
    from anakin_b200 import modelzoo
    graph, x, w32 = E.exact_walk(name, batch, "fp32")
    _, _, w16 = E.exact_walk(name, batch, "fp16")
    G = _graph(graph, name, batch)
    head = modelzoo.HEAD_DENSE[name]
    report = []
    nets = {}
    # the FP16 Net first: the fold cache it fills is the one the FP32 Net of the same Graph then reuses
    for prec, wk in (("fp16", w16), ("fp32", w32)):
        twin = api.Net(G, prec, keep_edges=True)
        _run(twin, x)
        edges, elems = _check_edges(twin, graph, wk, "%s b%d %s" % (name, batch, prec))
        # the probabilities against float64 within the kernel's derived bound
        prob = twin.get_output()
        logits = wk.vals[head].reshape(batch, -1).astype(np.float64)
        bound = softmax_bound(logits, rows_adds(logits.shape[1]))
        assert (np.abs(prob - wk.prob) <= bound).all(), (name, batch, prec, float(np.abs(prob - wk.prob).max()))
        # a default Net (shared buffers, CUDA graph, side stream): the twin's bits, over two predictions
        plain = api.Net(G, prec)
        _run(plain, x, times=2)
        assert plain.cuda_graph_active()
        for got, want in ((plain.get_output(), prob), (plain.read_tensor(head)[0], twin.read_tensor(head)[0])):
            assert np.array_equal(_bits(got), _bits(want)), (name, batch, prec, "default Net")
        nets[prec] = twin
        report.append("%s %d edges, %d values" % (prec, edges, elems))
    # FP16 and FP32 agree wherever the fp16 walk did not round
    same = 0
    for op_name, op in nets["fp16"].exec_order():
        if op == "Softmax":
            continue
        node = _pooled_by(graph, op_name) if op.endswith("Pool") else op_name
        v16, v32 = w16.vals[node], w32.vals[node]
        keep = v16.astype(np.float32) == v32
        a16 = _valid(*nets["fp16"].read_tensor(op_name), v16.shape).astype(np.float32)
        a32 = _valid(*nets["fp32"].read_tensor(op_name), v32.shape).astype(np.float32)
        assert np.array_equal(a16[keep], a32[keep]), (name, batch, op_name)
        same += int(keep.sum())
    assert same > 0
    print("%s b%d: %s; fp16 == fp32 on %d values" % (name, batch, ", ".join(report), same))
