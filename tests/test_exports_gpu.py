"""GPU: interior-tensor exports (Net(..., exports=[...]), Worker(..., exports=[...]), b200_export_run). Every
comparison is bit for bit: an export is the fp32 NCHW value of its edge tensor -- 8-bit codes x scale (x 127/255 for
uint8 codes) as oracle/model_walker.py's as_float, f16 widened, f32 copied -- and adding exports changes nothing else
about the net: exec order, activation bytes, fused head and outputs."""
import functools
import os
import tempfile

import numpy as np
import pytest

import pil_resize_oracle as P

pytestmark = pytest.mark.gpu

U8_FACTOR = np.float32(127.0 / 255.0)
CASES = {"tiny_resnet": (4, 32), "tiny_mobilenet": (4, 32), "resnet50": (8, 224)}


def _graph(name, batch, precision):
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build(name, batch=batch, precision=precision)
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return g, G


def _as_float(arr, dtype, scale):
    """oracle/model_walker.py as_float on codes (dtype 3 INT8, 7 UINT8) or float values."""
    if dtype in (3, 7):
        v = arr.astype(np.float32) * np.float32(scale)
        return v * U8_FACTOR if dtype == 7 else v
    return arr.astype(np.float32)


def _nchw(v_nhwc, n):
    return np.ascontiguousarray(np.transpose(v_nhwc, (0, 3, 1, 2))) if v_nhwc.ndim == 4 else v_nhwc.reshape(n, -1, 1, 1)


def _decode_edge(net, node):
    """The fp32 NCHW value of a keep_edges net's raw edge tensor."""
    arr, info = net.read_tensor(node)
    n, c, h, w = info["dims"]
    return _nchw(_as_float(arr[..., :c].reshape(n, h, w, c), info["dtype"], info["scale"]), n)


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _interior_nodes(net):
    """Every launched op whose tensor is not a graph output."""
    outs = {net.device_ptr(o) for o in net.out_names}
    return [n for n, _ in net.exec_order() if net.device_ptr(n) not in outs]


def _run(net, x, times=1):
    for _ in range(times):
        net.set_input("input_0", x)
        net.prediction()
    net.sync()


@functools.lru_cache(maxsize=None)
def _oracle(name):
    from anakin_b200 import modelzoo
    from oracle import model_walker as W
    batch, hw = CASES[name]
    g, _ = _graph(name, batch, "int8")
    x = modelzoo.synthetic_input(batch, hw)
    scales = {k: float(np.float32(v)) for k, v in modelzoo.load_calibration(name).items()}
    want, trace = W.run_int8(g, x, scales, return_intermediate=True)
    return x, want, trace


def _oracle_value(trace, node, op, n):
    # a conv that absorbed its MAX pooling holds the pooled tensor, which the oracle names pool1
    arr, dt, sc = trace["pool1" if op.endswith("Pool") else node]
    return _nchw(_as_float(arr, dt, sc), n)


# ---------------------------------------------------------------------------------------------- 1, 2. INT8
@pytest.mark.parametrize("name,cuda_graph", [("tiny_resnet", True), ("tiny_resnet", False), ("tiny_mobilenet", True),
                                             ("resnet50", True), ("resnet50", False)])
def test_int8_every_tensor_exported_at_once(name, cuda_graph):
    """Every launched op's output in one Net with buffer sharing on, against the oracle and a keep_edges twin."""
    from anakin_b200 import api
    batch, _ = CASES[name]
    x, want, trace = _oracle(name)
    _, G = _graph(name, batch, "int8")
    plain = api.Net(G, "int8")
    nodes = _interior_nodes(plain)
    net = api.Net(G, "int8", exports=nodes)
    if not cuda_graph:
        net.set_cuda_graph(False)
    assert net.export_names == nodes
    assert net.exec_order() == plain.exec_order()
    assert net.activation_bytes() == plain.activation_bytes() < net.activation_bytes_unshared()
    assert net.launched_ops() == plain.launched_ops() + len(nodes)
    assert net.export_bytes() == sum(4 * int(np.prod(net.export_info(n))) for n in nodes)
    _run(plain, x)
    _run(net, x, times=3)
    assert net.cuda_graph_active() == cuda_graph
    assert _same_bits(net.get_output(), plain.get_output())
    twin = api.Net(G, "int8", keep_edges=True)
    _run(twin, x)
    ops = dict(plain.exec_order())
    checked = 0
    for node in nodes:
        got = net.get_export(node, nchw=True)
        assert _same_bits(got, _decode_edge(twin, node)), (name, node)
        key = "pool1" if ops[node].endswith("Pool") else node
        if key in trace:
            assert _same_bits(got, _oracle_value(trace, node, ops[node], batch)), (name, node, ops[node])
            checked += 1
    assert checked >= min(10, len(nodes) - 1), checked
    if name == "tiny_mobilenet":
        assert any(n.endswith("_dw") for n in nodes)
    assert (net.get_output().argmax(1) == want["prob_out"].argmax(1)).all()


# ---------------------------------------------------------------------------------------------- 3. FP16 / FP32
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("name", ["tiny_resnet", "tiny_mobilenet"])
def test_float_nets_exports_equal_the_twin(name, precision):
    from anakin_b200 import api, modelzoo
    batch, hw = CASES[name]
    _, G = _graph(name, batch, precision)
    x = modelzoo.synthetic_input(batch, hw, seed=7)
    plain = api.Net(G, precision)
    nodes = _interior_nodes(plain)
    net = api.Net(G, precision, exports=nodes)
    twin = api.Net(G, precision, keep_edges=True)
    for n_ in (plain, twin):
        _run(n_, x)
    _run(net, x, times=3)
    assert net.exec_order() == plain.exec_order() and net.activation_bytes() == plain.activation_bytes()
    assert _same_bits(net.get_output(), plain.get_output())
    dtypes = set()
    for node in nodes:
        dtypes.add(twin.tensor_info(node)["dtype"])
        assert _same_bits(net.get_export(node, nchw=True), _decode_edge(twin, node)), (name, precision, node)
    if precision == "fp16":
        assert 0 in dtypes, "an f16 edge must be exported"


# ---------------------------------------------------------------------------------------------- 4. side stream
def test_side_stream_export_and_alias():
    """The projection shortcut runs on the side stream (joined three ops later): exported alone it must hold its own
    values, not what a later op left in its shared buffer. An alias node (Split) exports its producer's tensor."""
    from anakin_b200 import api, modelzoo
    _, G = _graph("tiny_resnet", 4, "int8")
    x = modelzoo.synthetic_input(4, 32, seed=3)
    for node in ("res2a_branch1", "res3a_branch1"):
        net = api.Net(G, "int8", exports=[node, "pool1_split"])
        twin = api.Net(G, "int8", keep_edges=True)
        _run(net, x, times=3)
        _run(twin, x)
        assert net.cuda_graph_active()
        assert _same_bits(net.get_export(node, nchw=True), _decode_edge(twin, node)), node
        assert _same_bits(net.get_export("pool1_split", nchw=True), _decode_edge(twin, "conv1"))


# ---------------------------------------------------------------------------------------------- 5. fused head
def test_fused_head_stays_fused_with_pool5_and_fc_exported():
    from anakin_b200 import api
    x, want, trace = _oracle("resnet50")
    _, G = _graph("resnet50", 8, "int8")
    plain = api.Net(G, "int8")
    net = api.Net(G, "int8", exports=["pool5", "fc1000"])
    order = plain.exec_order()
    assert net.exec_order() == order
    assert plain.launched_ops() == len(order) - 2, "the INT8 head must be one launch"
    assert net.launched_ops() == len(order) - 2 + 2
    _run(plain, x)
    _run(net, x, times=3)
    assert _same_bits(net.get_output(), plain.get_output())
    pool5 = net.get_export("pool5")
    arr, dt, sc = trace["pool5"]
    assert dt == 7
    assert _same_bits(pool5, _as_float(arr, dt, sc).reshape(8, -1))
    assert pool5.shape == (8, 2048)
    logits = net.get_export("fc1000")
    assert logits.shape == (8, 1000)
    assert _same_bits(logits, trace["fc1000"][0].reshape(8, -1))
    assert (net.get_output().argmax(1) == want["prob_out"].argmax(1)).all()


# ---------------------------------------------------------------------------------------------- 6. image inputs
MEAN = [123.675, 116.28, 103.53]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375]


def test_resizing_image_input_exports_equal_the_fp32_input_net():
    from anakin_b200 import anakin_bin, api, modelzoo
    batch, S, H = 2, 36, 32
    g = modelzoo.build("tiny_resnet", batch=batch, precision="int8")
    blob = anakin_bin.dumps(g)
    Gf, Gi = api.Graph.from_bytes(blob), api.Graph.from_bytes(blob)
    Gi.set_input_image("input_0", MEAN, SCALE, [2, 1, 0])
    Gi.set_input_image_resize("input_0", 96, 96, S, filter="pil")
    for G_ in (Gf, Gi):
        G_.ResetBatchSize("input_0", batch)
        G_.Optimize()
    nodes = _interior_nodes(api.Net(Gf, "int8"))
    nf, ni = api.Net(Gf, "int8", exports=nodes), api.Net(Gi, "int8", exports=nodes)
    rng = np.random.default_rng(11)
    for it, sizes in enumerate([[(32, 32), (75, 41)], [(96, 17), (40, 90)], [(64, 64), (1, 1)]]):
        imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
        u8 = P.resize_batch(imgs, S, H, H)[..., [2, 1, 0]].astype(np.float32)
        x = (u8 - np.asarray(MEAN, np.float32)) * np.asarray(SCALE, np.float32)
        nf.set_input("input_0", np.ascontiguousarray(np.transpose(x, (0, 3, 1, 2))))
        ni.set_input_images("input_0", imgs)
        nf.prediction()
        ni.prediction()
        nf.sync(); ni.sync()
        for node in nodes:
            assert _same_bits(ni.get_export(node), nf.get_export(node)), (it, node)
        assert _same_bits(ni.get_output(), nf.get_output()), it
    assert ni.cuda_graph_active()


# ---------------------------------------------------------------------------------------------- 7. Worker
def test_worker_view_results_hold_output_and_exports():
    import torch
    from anakin_b200 import api, modelzoo
    batch, nreq = 4, 8
    g, G = _graph("tiny_resnet", batch, "int8")
    net = api.Net(G, "int8", exports=["pool5"])
    xs = [modelzoo.synthetic_input(batch, 32, seed=200 + i) for i in range(nreq)]
    want = []
    for x in xs:
        _run(net, x)
        out, info = net.read_tensor(net.out_names[0])
        want.append((out.reshape(-1).copy(), net.get_export("pool5").reshape(-1).copy()))
    n_out, n_pool = want[0][0].size, want[0][1].size
    with tempfile.TemporaryDirectory() as d:
        model = os.path.join(d, "tiny.anakin.bin")
        modelzoo.save(g, model)
        w = api.Worker(model, "int8", threads=2, devices=(0,), batch=batch, exports=["pool5"])
        assert w.output_count() == n_out + n_pool
        ins = [torch.from_numpy(x).pin_memory() for x in xs]
        outs = [torch.zeros(n_out + n_pool, dtype=torch.float32).pin_memory() for _ in range(nreq)]
        for rnd in range(2):
            for i in range(nreq):
                w.async_prediction_ptr(ins[i].data_ptr(), ins[i].numel(), outs[i].data_ptr(), outs[i].numel())
            for i in range(nreq):
                w.async_get_result()
            for i in range(nreq):
                parts = api.split_view(outs[i].numpy(), [("prob", (n_out,)), ("pool5", (batch, n_pool // batch))])
                assert _same_bits(parts["prob"], want[i][0]), (rnd, i)
                assert _same_bits(parts["pool5"].reshape(-1), want[i][1]), (rnd, i)
                outs[i].zero_()
        assert any((want[0][1] != want[i][1]).any() for i in range(1, nreq)), "inputs must differ for the order check"
        # a wrong out_count fails that request alone
        short = torch.zeros(n_out + n_pool - 1, dtype=torch.float32).pin_memory()
        w.async_prediction_ptr(ins[0].data_ptr(), ins[0].numel(), short.data_ptr(), short.numel())
        w.async_prediction_ptr(ins[1].data_ptr(), ins[1].numel(), outs[1].data_ptr(), outs[1].numel())
        with pytest.raises(api.AnakinError, match="out_count %d, the result is %d" % (n_out + n_pool - 1, n_out + n_pool)):
            w.async_get_result()
        w.async_get_result()
        assert _same_bits(outs[1].numpy()[n_out:], want[1][1])
        del w
        # an interior edge exports its bottom's tensor; an edge that does not exist fails creation
        w = api.Worker(model, "int8", threads=1, devices=(0,), batch=batch, exports=[("res3b_branch2c", "pool5")])
        assert w.output_count() == n_out + int(np.prod(net.tensor_info("res3b_branch2c")["dims"]))
        del w
        with pytest.raises(api.AnakinError, match="no edge pool5 -> fc7"):
            api.Worker(model, "int8", threads=1, devices=(0,), batch=batch, exports=[("pool5", "fc7")])


# ---------------------------------------------------------------------------------------------- 8. refusals
@pytest.mark.parametrize("exports,message", [
    (["nope"], "export nope: no node of that name in the optimised graph"),
    (["bn_conv1"], "export bn_conv1: no node of that name"),
    (["input_0"], "export input_0: is a graph input"),
    (["pool5", "fc", "pool5"], "export pool5: registered twice"),
    (["prob"], "export prob: is a graph output"),
    (["prob_out"], "export prob_out: is a graph output"),
])
def test_refusals(exports, message):
    from anakin_b200 import api
    _, G = _graph("tiny_resnet", 2, "int8")
    with pytest.raises(api.AnakinError, match=message):
        api.Net(G, "int8", exports=exports)
