"""GPU: the shared activation memory of every net against the launches that actually run.

With buffer sharing on (the default), NetCore::plan_activation_memory hands a tensor's buffer to another tensor once
its last reader is issued. Whether two tensors land in one buffer depends on the net, the batch and the precision,
and a race between them shows in the outputs only sometimes, so comparing outputs can miss it. The static audit here
(tests/activation_plan.py) derives every tensor's live steps from the launch rules of NetCore::run_eager and
Net.schedule() -- main stream, side stream up to its join, the fused head over the steps of the three ops it covers --
and checks the device pointers of a constructed Net against them. It never runs a prediction.

Programmatic dependent launch is assumed to touch only weights before a kernel's grid-dependency wait; under that
assumption a launch occupies its own step only. The audit does not test the assumption.

The poisoned runs then fill every shared buffer with 0xFF bytes (NaN in float edges) before the first prediction and
between CUDA-graph replays: outputs, exports and calibration maxima must stay bit-identical to a keep_edges twin, so
no kernel reads bytes of its buffer that nothing wrote in the current pass."""
import functools
import os

import numpy as np
import pytest

from activation_plan import plan_of, violations

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BATCHES = (1, 3, 8, 16)        # the fused INT8 head takes at most 8 images: 16 keeps the three head ops


def _precisions(name):
    """fp32 and fp16, and int8 where the zoo has a calibration table for the net."""
    has_table = os.path.exists(os.path.join(GOLD, "%s_calib.json" % name))
    return ("fp32", "fp16", "int8") if has_table else ("fp32", "fp16")


def _zoo():
    from anakin_b200 import modelzoo
    return sorted(modelzoo.BUILDERS)


@functools.lru_cache(maxsize=None)
def _blob(name, precision):
    from anakin_b200 import anakin_bin, modelzoo
    return anakin_bin.dumps(modelzoo.build(name, batch=1, precision=precision))


def _graph_of(blob, batch):
    from anakin_b200 import api
    G = api.Graph.from_bytes(blob)
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return G


def _graph(name, precision, batch):
    return _graph_of(_blob(name, precision), batch)


def _audit(G, precision, **kw):
    """(net, plan) of a Net built with buffer sharing on, after asserting the audit finds nothing."""
    from anakin_b200 import api
    net = api.Net(G, precision, **kw)
    plan = plan_of(net, G)
    found = violations(plan)
    assert not found, "\n".join(found)
    assert net.activation_bytes() < net.activation_bytes_unshared(), "no buffer is shared: the audit checked nothing"
    return net, plan


def _overlap(a, b):
    return a[0] < b[0] + b[1] and b[0] < a[0] + a[1]


# ---------------------------------------------------------------------------------------------- 1. every zoo net
CASES = [(n, p, b) for n in _zoo() for p in _precisions(n) for b in BATCHES]


@pytest.mark.parametrize("name,precision,batch", CASES, ids=["%s-%s-b%d" % c for c in CASES])
def test_shared_buffers_are_never_live_together(name, precision, batch):
    _audit(_graph(name, precision, batch), precision)


@pytest.mark.parametrize("name,precision", [(n, p) for n in _zoo() for p in _precisions(n)])
def test_keep_edges_shares_nothing(name, precision):
    from anakin_b200 import api
    G = _graph(name, precision, 3)
    net = api.Net(G, precision, keep_edges=True)
    found = violations(plan_of(net, G), keep_edges=True)
    assert not found, "\n".join(found)
    assert net.activation_bytes() == net.activation_bytes_unshared()


# ---------------------------------------------------------------------------------------------- 2. variants
@pytest.mark.parametrize("name,precision,batch", [("mobilenet_v1", "int8", 8), ("vgg16", "fp16", 3)])
def test_without_the_side_stream(name, precision, batch):
    """A chain without off-chain ops runs on the main stream alone."""
    net, _ = _audit(_graph(name, precision, batch), precision)
    assert all(e["join"] is None for e in net.schedule())


@pytest.mark.parametrize("name,batch", [("mobilenet_v1", 9), ("resnet50", 12), ("tiny_resnet", 16)])
def test_without_the_fused_head(name, batch):
    """Above 8 images plan_fused_head declines: the INT8 head runs as its three ops."""
    net, _ = _audit(_graph(name, "int8", batch), "int8")
    assert all(e["head"] == 0 for e in net.schedule())


@pytest.mark.parametrize("name,batch", [("resnet50", 3), ("tiny_resnet", 8)])
def test_fp32_with_calibration_statistics(name, batch):
    net, _ = _audit(_graph(name, "fp32", batch), "fp32", calib_stats=True)
    assert len(net.calib_names()) == 1 + len(net.exec_order())


@pytest.mark.parametrize("batch", [3, 8])
def test_int8_resnet_with_a_side_op_and_the_logits_exported(batch):
    net, _ = _audit(_graph("resnet50", "int8", batch), "int8", exports=["res3a_branch1", "fc1000"])
    sched = {e["name"]: e for e in net.schedule()}
    assert sched["res3a_branch1"]["join"] is not None and sched["fc1000"]["head"] == 2
    assert net.export_names == ["res3a_branch1", "fc1000"]


# ---------------------------------------------------------------------------------------------- 3. the report itself
INT8_RESNETS = ["tiny_resnet", "resnet50", "resnet101", "tiny_se_resnet", "se_resnet50"]


@pytest.mark.parametrize("name", INT8_RESNETS)
def test_side_ops_join_at_their_first_reader(name):
    from anakin_b200 import api
    G = _graph(name, "int8", 8)
    net = api.Net(G, "int8")
    plan = plan_of(net, G)
    side = [(i, e) for i, e in enumerate(plan.ops) if e["join"] is not None]
    assert side, "an INT8 ResNet runs its projection shortcuts on the side stream"
    for i, e in side:
        readers = [k for k, o in enumerate(plan.ops) if e["name"] in plan.reads[o["name"]]]
        assert e["name"].endswith("_branch1") and readers and readers[0] == e["join"], (e, readers)
        assert all(o["join"] is None for o in plan.ops[i + 1:e["join"] + 1]), "side ops do not overlap"


@pytest.mark.parametrize("name", [n for n in _zoo() if "int8" in _precisions(n)])
def test_int8_heads_are_fused_up_to_eight_images(name):
    from anakin_b200 import api
    for batch in BATCHES:
        net = api.Net(_graph(name, "int8", batch), "int8")
        sched = net.schedule()
        head = [(e["op"], e["head"]) for e in sched if e["head"]]
        if batch <= 8:
            assert head == [("Pooling", 1), ("Dense", 2), ("Softmax", 2)], (batch, head)
            assert [e["head"] for e in sched[-3:]] == [1, 2, 2]
            assert net.launched_ops() == len(sched) - 2
        else:
            assert head == [], (batch, head)
            assert net.launched_ops() == len(sched)


# ---------------------------------------------------------------------------------------------- 4. the head's input
def _head_tensors(plan):
    head = [e["name"] for e in plan.ops if e["head"]]
    assert len(head) == 3, "the INT8 head is not fused"
    return plan.reads[head[0]][0], head[1]          # the pooling input, the logits


@pytest.mark.parametrize("batch", [1, 8])
def test_mobilenet_v1_int8_logits_stay_out_of_the_heads_input(batch):
    """A net without branches alternates between two buffers: at the logits' step the pooling input's buffer is the
    only free one unless the memory plan knows that the fused head still pools that input while it stores logits."""
    _, plan = _audit(_graph("mobilenet_v1", "int8", batch), "int8")
    pooled_in, logits = _head_tensors(plan)
    assert (pooled_in, logits) == ("conv14_sep", "fc7")
    assert not _overlap(plan.tensors[pooled_in], plan.tensors[logits])


def _chain_blob(batch):
    """conv -> conv -> global average pool -> fc (1000 outputs) -> softmax, INT8."""
    from anakin_b200 import anakin_bin, modelzoo
    g = modelzoo.GraphBuilder("HeadChain", seed=5)
    x = g.input("input_0", (batch, 3, 32, 32))
    x = g.relu("conv1_relu", g.conv("conv1", x, 3, 32, 3, 2, 1, bias=True))
    x = g.relu("conv2_relu", g.conv("conv2", x, 32, 1024, 3, 2, 1, bias=True))
    x = g.pool("pool", x, 8, 1, 0, "AVG", global_pooling=True)
    x = g.softmax("prob", g.dense("fc", x, 1024, 1000))
    g.output("prob_out", x)
    graph = g.finalize()
    scales = {"input_0": 1 / 127, "conv1": 0.02, "conv1_relu": 0.02, "conv2": 0.03, "conv2_relu": 0.03,
              "pool": 0.01, "fc": 0.02, "prob": 1 / 127}
    return anakin_bin.dumps(modelzoo.apply_int8(graph, scales))


@pytest.mark.parametrize("batch", [1, 8])
def test_hand_built_head_chain_keeps_its_input(batch):
    G = _graph_of(_chain_blob(batch), batch)
    _, plan = _audit(G, "int8")
    pooled_in, logits = _head_tensors(plan)
    assert (pooled_in, logits) == ("conv2", "fc")
    assert not _overlap(plan.tensors[pooled_in], plan.tensors[logits])


# ---------------------------------------------------------------------------------------------- 5. poisoned buffers
class _Span:
    """`n` device bytes at `ptr`, for torch.as_tensor."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "strides": None,
                                        "version": 2}


def _shared_spans(plan):
    """The byte ranges of the shared buffers: every tensor that is not a graph input, a graph output or padded, merged
    where they overlap."""
    spans = sorted((p, p + n) for t, (p, n, padded) in plan.tensors.items()
                   if n and not padded and t not in plan.pinned)
    merged = []
    for lo, hi in spans:
        if merged and lo < merged[-1][1]:
            merged[-1][1] = max(merged[-1][1], hi)
        else:
            merged.append([lo, hi])
    return merged


def _poison(spans):
    import torch
    for lo, hi in spans:
        torch.as_tensor(_Span(lo, hi - lo), device="cuda").fill_(0xFF)
    torch.cuda.synchronize()


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


POISON = [("mobilenet_v1", "int8", 8, False), ("resnet50", "int8", 8, False), ("tiny_se_resnet", "fp16", 4, False),
          ("tiny_resnet", "fp32", 4, True)]


@pytest.mark.parametrize("name,precision,batch,calib", POISON, ids=["%s-%s-b%d" % c[:3] for c in POISON])
def test_poisoned_shared_buffers_change_nothing(name, precision, batch, calib):
    import torch
    from anakin_b200 import api, modelzoo
    torch.cuda.init()
    G = _graph(name, precision, batch)
    plain = api.Net(G, precision)
    interior = [e["name"] for e in plain.schedule() if e["name"] not in plan_of(plain, G).pinned]
    del plain
    net, plan = _audit(G, precision, calib_stats=calib, exports=interior)
    twin = api.Net(G, precision, keep_edges=True, calib_stats=calib, exports=interior)
    x = modelzoo.synthetic_input(batch, G.input_shape("input_0")[2], seed=9)
    twin.set_input("input_0", x)
    twin.prediction()
    twin.sync()
    want = {n: twin.get_export(n, nchw=True) for n in interior}
    spans = _shared_spans(plan)
    # every shared buffer is filled: activation_bytes() less the tensors that keep a buffer of their own
    assert sum(hi - lo for lo, hi in spans) == net.activation_bytes() - sum(
        n for t, (_, n, padded) in plan.tensors.items() if padded or t in plan.pinned)
    net.set_input("input_0", x)
    for run in range(3):        # eager, captured into a CUDA graph, replayed
        _poison(spans)
        net.prediction()
        net.sync()
        assert _same_bits(net.get_output(), twin.get_output()), (name, run)
        for n in interior:
            assert _same_bits(net.get_export(n, nchw=True), want[n]), (name, run, n)
        if calib:
            assert _same_bits(net.calib_read(hist=False)[0], twin.calib_read(hist=False)[0]), (name, run)
    assert net.cuda_graph_active()
