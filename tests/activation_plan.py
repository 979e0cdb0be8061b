"""Audit of a Net's shared activation memory against the launches that run.

The live range of every edge tensor is derived from the launch rules of NetCore::run_eager, not from the memory
planner's own bookkeeping, in steps = indices of Net.exec_order():
  * an op on the main stream occupies its own step k;
  * a side-stream op i joined at j (Net.schedule) occupies steps i .. j - 1: it is forked behind op i - 1 and may run
    next to the main ops up to j - 1; its reader j waits for it;
  * the fused head (head 1 at the pooling op, head 2 at the inner product and the softmax it covers) occupies the
    pooling op's step through the softmax's: over all of them it reads the pooling input and writes the pooled rows,
    the logits and the probabilities;
  * exports and calibration statistics read a tensor in its producer's steps (on the producer's stream, before its
    first reader), so they extend no live range.
A tensor is live from the first step of its producer to the last step of its last reader. Two tensors whose byte
ranges [ptr, ptr + bytes) overlap must never be live at the same step. Graph inputs and outputs (read and written by
the user between predictions) and NHWC tensors with channel padding (whose padding is never written and must stay 0)
may overlap nothing at all.

Programmatic dependent launch lets a kernel start while its predecessor in the stream is still running; this audit
assumes that every kernel touches only its weights before its grid-dependency wait, so that a launch occupies its own
step only.

`plan_of(net, graph)` reads a Net's plan through the C API without running it; `violations(plan)` is pure Python.
"""
import collections

Plan = collections.namedtuple("Plan", "ops reads tensors pinned")
# ops: [{"name", "op", "join", "head"}] (Net.schedule); reads: {op name: [tensor names]}; tensors: {tensor name:
# (ptr, bytes, padded)}, a tensor being named by its producing node; pinned: {tensor name: "graph input" | ...}.

ALIAS_OPS = ("Split", "Flatten", "Gather", "Output")


def occupancy(ops):
    """[(first, last)] steps of every op of the schedule."""
    occ = [None] * len(ops)
    for k, e in enumerate(ops):
        if e["head"] == 1:
            end = k
            while end + 1 < len(ops) and ops[end + 1]["head"] == 2:
                end += 1
            for i in range(k, end + 1):
                occ[i] = (k, end)
        elif e["head"] == 2:
            assert occ[k] is not None, "op %s is covered by a fused head that does not launch before it" % e["name"]
        elif e["join"] is not None:
            assert e["join"] > k + 1, "side op %s joined at %d" % (e["name"], e["join"])
            occ[k] = (k, e["join"] - 1)
        else:
            occ[k] = (k, k)
    return occ


def live_ranges(plan):
    """{tensor name: (first step, last step)} of every tensor some op writes or reads."""
    occ = occupancy(plan.ops)
    live = {}

    def touch(t, steps):
        lo, hi = live.get(t, steps)
        live[t] = (min(lo, steps[0]), max(hi, steps[1]))

    for k, e in enumerate(plan.ops):
        touch(e["name"], occ[k])
        for t in plan.reads.get(e["name"], ()):
            touch(t, occ[k])
    return live


def violations(plan, keep_edges=False):
    """Human-readable list of every pair of tensors the plan puts in one place while both are live (keep_edges: any
    two tensors in one place), and of every pinned or padded tensor that shares bytes with another."""
    live = live_ranges(plan)
    names = sorted((t for t, (ptr, nbytes, _) in plan.tensors.items() if nbytes > 0), key=lambda t: plan.tensors[t][0])
    out = []
    for t in names:
        if not plan.tensors[t][0]:
            out.append("%s has %d bytes and no device pointer" % (t, plan.tensors[t][1]))
    for i, a in enumerate(names):
        pa, na, pad_a = plan.tensors[a]
        for b in names[i + 1:]:
            pb, nb, pad_b = plan.tensors[b]
            if pb >= pa + na:
                break       # sorted by ptr: no later tensor starts inside a
            why = "%s [%#x, +%d) and %s [%#x, +%d) share bytes" % (a, pa, na, b, pb, nb)
            if keep_edges:
                out.append(why + " with keep_edges=True")
                continue
            special = [(t, plan.pinned.get(t) or "padded") for t, pad in ((a, pad_a), (b, pad_b))
                       if t in plan.pinned or pad]
            if special:
                out.append(why + "; %s may share nothing" % ", ".join("%s (%s)" % s for s in special))
                continue
            la, lb = live.get(a), live.get(b)
            if la is None or lb is None:
                out.append(why + "; %s is never written or read" % (a if la is None else b))
            elif la[0] <= lb[1] and lb[0] <= la[1]:
                out.append(why + " while both are live: %s in steps %d..%d (%s .. %s), %s in steps %d..%d (%s .. %s)"
                           % (a, la[0], la[1], plan.ops[la[0]]["name"], plan.ops[la[1]]["name"],
                              b, lb[0], lb[1], plan.ops[lb[0]]["name"], plan.ops[lb[1]]["name"]))
    return out


def plan_of(net, graph):
    """The Plan of a constructed Net (api.Net) of the optimised api.Graph `graph`: schedule, the tensors each op
    reads (graph.describe(), alias nodes resolved to their producer), and every tensor's bytes and device pointer."""
    ops = net.schedule()
    launched = {e["name"] for e in ops}
    nodes = {name: (op, ins) for name, op, ins, _ in graph.describe()}

    def producer(name):
        seen = name
        while name not in launched and nodes[name][0] != "Input":
            op, ins = nodes[name]
            assert op in ALIAS_OPS and ins, "%s (%s) is neither launched nor an alias" % (name, op)
            name = ins[0]
        # an alias returns its producer's pointer
        assert net.device_ptr(seen) == net.device_ptr(name), (seen, name)
        return name

    reads = {e["name"]: [producer(b) for b in nodes[e["name"]][1]] for e in ops}
    tensors = {}
    for name, (op, _) in nodes.items():
        if name in launched or op == "Input":
            info = net.tensor_info(name)
            padded = info["layout"] == 9 and info["c_stored"] != info["dims"][1]
            tensors[name] = (net.device_ptr(name) or 0, info["bytes"], padded)
    pinned = {producer(n): "graph input" for n in net.in_names}
    pinned.update({producer(n): "graph output" for n in net.out_names})
    return Plan(ops, reads, tensors, pinned)
