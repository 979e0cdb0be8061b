"""The designed nets of net_exact.py on the CPU: the walk's invariants at every net, shape and batch the GPU test uses,
the exact FP32 walk against the model-level oracle bit for bit, and negative controls showing that the designed data
would catch the framework bugs the GPU test is there for."""
import numpy as np
import pytest

import net_exact as E
from test_net_exact_gpu import CASES

BIG = sorted({n for n, _ in CASES} - {"tiny_resnet", "tiny_mobilenet"})


def _bits(a):
    a = np.where(a == 0, np.zeros((), a.dtype), a).astype(a.dtype)
    return a.view(np.uint16 if a.dtype == np.float16 else np.uint32)


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("name,batch", [c for c in CASES if c[0] not in BIG] + [(n, 1) for n in BIG])
def test_walk_invariants(name, batch, precision):
    """exact_walk asserts every sum's exactness and the data's density as it goes (big nets at batch 1 here)."""
    _, _, wk = E.exact_walk(name, batch, precision)
    assert wk.stats["sums"] > 0 and wk.stats["max_bits"] <= E.EXACT_BITS


@pytest.mark.parametrize("name,batch", [("tiny_resnet", 3), ("tiny_mobilenet", 3), ("resnet50", 1),
                                        ("mobilenet_v1", 1)])
def test_fp32_walk_equals_oracle(name, batch, oracle):
    """On exact sums fp32 re-association is irrelevant: model_walker.run_fp32 (its own grouping, the fold of
    parameter_fusion.cpp, the NCHW flatten) gives the walk's bits on every edge but the softmax."""
    from oracle import model_walker as MW
    graph, x, wk = E.exact_walk(name, batch, "fp32")
    _, vals = MW.run_fp32(graph, x, return_values=True)
    compared = 0
    for node, v in wk.vals.items():
        if graph_op(graph, node) in ("Softmax", "Output", "Input"):
            continue
        want = np.asarray(vals[node], np.float32).reshape(v.shape)
        assert np.array_equal(_bits(v), _bits(want)), "%s: %s differs from the oracle" % (name, node)
        compared += 1
    assert compared >= 10


def graph_op(graph, node):
    return next(n["op"] for n in graph["nodes"] if n["name"] == node)


MUTATIONS = {
    "no_eps": ("tiny_resnet", "fp32"),
    "f16_before_fold": ("tiny_resnet", "fp16"),
    "avg_counts_padding": ("tiny_resnet", "fp32"),
    "nhwc_flatten": ("vgg16", "fp32"),
    "residual_other": ("tiny_resnet", "fp16"),
    "swap_tail": ("tiny_mobilenet", "fp16"),
}


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_negative_controls(mutation):
    """Each bug, restated as a mutation of the walk, changes at least one compared edge of a designed net."""
    name, precision = MUTATIONS[mutation]
    batch = 1 if name == "vgg16" else 3
    graph, x, wk = E.exact_walk(name, batch, precision)
    bad = E.walk(graph, x, precision, mutate=(mutation,), check=False)
    changed = [n for n, v in wk.vals.items() if graph_op(graph, n) not in ("Softmax", "Output")
               and not np.array_equal(_bits(v), _bits(np.asarray(bad.vals[n], v.dtype)))]
    assert changed, "%s changes no edge of %s %s" % (mutation, name, precision)
