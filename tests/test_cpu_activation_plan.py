"""CPU suite: the activation-plan audit (tests/activation_plan.py) on hand-written plans. It must reject the plan the
memory planner made before it knew about the fused head -- the logits in the buffer of the head's input -- and
accept the same buffers when the three head ops run one after another."""
from activation_plan import Plan, violations

MB = 1 << 20


def _chain(head, logits_at):
    """input -> conv_a -> conv_b -> pool -> fc -> prob, buffers X / Y alternating as a best-fit planner hands them
    out; the logits (fc) at `logits_at`."""
    X, Y, P, IN = 0x10000000, 0x20000000, 0x30000000, 0x40000000
    ops = [{"name": n, "op": o, "join": None, "head": h} for n, o, h in (
        ("conv_a", "ConvRelu", 0), ("conv_b", "ConvRelu", 0), ("pool", "Pooling", head),
        ("fc", "Dense", 2 if head else 0), ("prob", "Softmax", 2 if head else 0))]
    reads = {"conv_a": ["input_0"], "conv_b": ["conv_a"], "pool": ["conv_b"], "fc": ["pool"], "prob": ["fc"]}
    tensors = {"input_0": (IN, MB, False), "conv_a": (X, MB, False), "conv_b": (Y, MB, False),
               "pool": (X, 8192, False), "fc": (logits_at, 32000, False), "prob": (P, 32000, False)}
    return Plan(ops, reads, tensors, {"input_0": "graph input", "prob": "graph output"})


def test_logits_in_the_fused_heads_input_are_rejected():
    found = violations(_chain(head=1, logits_at=0x20000000))
    assert len(found) == 1, found
    assert "conv_b" in found[0] and "fc" in found[0] and "while both are live" in found[0]
    assert "steps 1..4" in found[0] and "steps 2..4" in found[0], found[0]


def test_the_same_buffers_are_fine_for_three_separate_head_ops():
    assert violations(_chain(head=0, logits_at=0x20000000)) == []
    assert violations(_chain(head=1, logits_at=0x50000000)) == []


def test_keep_edges_allows_no_sharing_at_all():
    found = violations(_chain(head=0, logits_at=0x20000000), keep_edges=True)
    assert len(found) == 2 and all("keep_edges" in f for f in found), found     # conv_a / pool, conv_b / fc


def test_pinned_and_padded_tensors_share_nothing():
    p = _chain(head=0, logits_at=0x40000000 + 4096)         # inside the graph input
    found = violations(p)
    assert len(found) == 1 and "input_0 (graph input)" in found[0], found
    p = _chain(head=0, logits_at=0x50000000)
    p.tensors["fc"] = (0x10000000 + 16384, 32000, True)      # padded logits in conv_a's (dead) buffer, past pool
    found = violations(p)
    assert len(found) == 1 and "fc (padded)" in found[0], found


def test_a_side_op_is_live_until_its_join():
    """branch1 runs on the side stream from step 1 and is joined at step 4: the main ops 2 and 3 run next to it, so
    none of their outputs may take its buffer, and its input lives until step 3."""
    ops = [{"name": n, "op": "Conv", "join": j, "head": 0} for n, j in
           (("stem", None), ("branch1", 4), ("branch2a", None), ("branch2b", None), ("sum", None))]
    reads = {"stem": ["input_0"], "branch1": ["stem"], "branch2a": ["stem"], "branch2b": ["branch2a"],
             "sum": ["branch1", "branch2b"]}
    tensors = {"input_0": (0x1000, 64, False), "stem": (0x2000, 64, False), "branch1": (0x3000, 64, False),
               "branch2a": (0x4000, 64, False), "branch2b": (0x5000, 64, False), "sum": (0x6000, 64, False)}
    plan = Plan(ops, reads, tensors, {"input_0": "graph input", "sum": "graph output"})
    assert violations(plan) == []
    tensors["branch2b"] = (0x3000, 64, False)                # written at step 3, while branch1 may still run
    found = violations(plan)
    assert len(found) == 1 and "branch1" in found[0] and "branch2b" in found[0], found
    tensors["branch2b"] = (0x2000, 64, False)                # stem is still read by branch1 at step 3
    found = violations(plan)
    assert len(found) == 1 and "stem in steps 0..3" in found[0], found
