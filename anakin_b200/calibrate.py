"""INT8 calibration through the product's own FP32 path (Net<NV, FP32> on the GPU).

Mirrors the reference's calibration tooling:
  Calibrator / EntropyCalibrator    framework/core/net/calibrator.h:35-86, entropy_calibrator.cpp:24-369
  BatchStream                        framework/core/net/batch_stream.h
  the table file "<tensor name> <scale>" per line   entropy_calibrator.cpp:167-177 (write_calibrator)

Two passes over the calibration batches, as the reference makes them (get_max_values, then get_histgrams): the maximum
|x| of every tensor, then a 2048-bin histogram of |x| with bin width max / 2048. Scales:
  algo "maxabs"   scale = max / 127. This is what the reference's EntropyCalibrator EFFECTIVELY writes: its
                  get_kl_threshold computes the KL-optimal bin but inserts max / (127 * 2048) * 2048 (the `* thresh`
                  line is commented out, entropy_calibrator.cpp:348-349) -- and what CalibrationAlgoType::MAXABS means.
  algo "entropy"  scale = max / (127 * 2048) * thresh, thresh = the bin that minimises the KL divergence between the
                  clipped reference distribution and its 128-level quantisation -- the restated search of
                  entropy_calibrator.cpp:24-130,300-346 (the variant the reference left commented out).

The tensors observed are the outputs of the OPTIMISED graph's nodes (what the INT8 net requantises); every original
node a fused node absorbed (BatchNorm, Scale, ReLU, the Eltwise of a ConvEltwise, a fused MAX pooling) receives the
fused node's scale, so the table can be applied to the un-fused graph (modelzoo.apply_int8) exactly like the tables
under tests/golden/.

The statistics are computed on the GPU: the FP32 net is built with calib_stats=True, so every prediction runs
b200_calib_stats_run right behind each tensor's producer, inside the captured CUDA graph (the maxima of pass 1 bit for
bit, the histograms of pass 2 as equal integer arrays), and the entropy thresholds come from b200_calib_kl_run over all
histograms at once. Only the maxima and the 2048 counters per tensor reach the host. kl_threshold and its helpers below
are the specification that kernel is held to (tests/test_cpu_calibrate.py, tests/test_calibrate_gpu.py).
"""
import math

import numpy as np

from . import anakin_bin, api

BIN_NUM = 2048
QUANT_LEVELS = 128

_FUSABLE_FOLLOWERS = {"BatchNorm", "Scale", "ReLU", "Pooling", "Eltwise"}


class BatchStream:
    """Iterable source of fp32 NCHW calibration batches (batch_stream.h): a list / generator factory."""

    def __init__(self, batches):
        self._batches = batches

    def reset(self):
        return iter(self._batches() if callable(self._batches) else self._batches)


# ------------------------------------------------------------------------------------------------- KL threshold
def _get_ref_q(ref_p, q_size):
    """entropy_calibrator.cpp:36-55: shrink ref_p to q_size bins (partial bins weighted by their overlap; the counts
    are accumulated in an int, as there)."""
    p_size = len(ref_p)
    step = np.float32(p_size) / np.float32(q_size)
    ref_q = np.zeros(q_size, np.float32)
    for i in range(q_size):
        start, end = np.float32(step * i), np.float32(step * (i + 1))
        s_i, e_i, s_c = int(math.floor(start)), int(math.floor(end)), int(math.ceil(start))
        count = int(ref_p[s_c:e_i].sum())
        count = int(count + (s_c - start) * ref_p[s_i])
        if e_i < p_size:
            count = int(count + (end - e_i) * ref_p[e_i])
        ref_q[i] = count
    return ref_q


def _expand_to_q(ref_p, ref_q):
    """entropy_calibrator.cpp:58-95: spread every quantised bin over the non-empty source bins it covers."""
    q = np.zeros(len(ref_p), np.float32)
    coeff = np.float32(len(q)) / np.float32(len(ref_q))
    n = len(ref_p)
    for i in range(len(ref_q)):
        start, end = np.float32(i * coeff), np.float32((i + 1) * coeff)
        s_c, e_f, s_f = int(math.ceil(start)), int(math.floor(end)), int(math.floor(start))
        zero_num = float(np.count_nonzero(ref_p[s_c:e_f] == 0))
        if ref_p[s_f] == 0:
            zero_num += s_c - start
        if e_f < n and ref_p[e_f] == 0:
            zero_num += end - e_f
        dis = coeff - zero_num
        if dis <= 0:
            continue
        if ref_p[s_f] != 0:
            q[s_f] += (s_c - start) / dis * ref_q[i]
        nz = np.nonzero(ref_p[s_c:e_f])[0] + s_c
        q[nz] += np.float32(1.0) / dis * ref_q[i]
        if e_f < n and ref_p[e_f] != 0:
            q[e_f] += (end - e_f) / dis * ref_q[i]
    return q


def _kl_divergence(hist, q):
    """entropy_calibrator.cpp:99-128: KL(hist || q), the last bin of q spread over the tail of hist. hist is the FULL
    histogram (the reference passes `hist`, not the clipped ref_p)."""
    sum_p = float(hist.sum())
    sum_q = float(int(q.sum()))
    if sum_p <= 0 or sum_q <= 0:
        return float("inf")
    nq = len(q)
    p_prob = hist / sum_p
    q_prob = q / sum_q
    head = (hist[:nq - 1] != 0) & (q[:nq - 1] != 0)
    kl = float(np.sum(p_prob[:nq - 1][head] * np.log2(p_prob[:nq - 1][head] / q_prob[:nq - 1][head])))
    tail_q = float(q[nq - 1]) / sum_q / (len(hist) - nq + 1)
    tail = hist[nq - 1:] > 0
    if tail.any():
        if tail_q <= 0:
            return float("inf")
        kl += float(np.sum(p_prob[nq - 1:][tail] * np.log2(p_prob[nq - 1:][tail] / tail_q)))
    return kl


def kl_threshold(hist):
    """entropy_calibrator.cpp:300-346: the bin count (129 .. BIN_NUM - 2) whose clipped distribution, quantised to 128
    levels, is closest (KL) to the histogram. hist: int array of BIN_NUM bins of |x|."""
    hist = np.asarray(hist, np.int64)
    assert hist.shape == (BIN_NUM,)
    total = int(hist.sum() - hist[0])
    start_num = int(hist[1:129].sum())
    best, thresh = float("inf"), 0
    for i in range(129, BIN_NUM - 1):
        ref_p = hist[1:i + 1].copy()
        ref_p[i - 1] += total - start_num          # the outliers join the last kept bin
        ref_q = _get_ref_q(ref_p, QUANT_LEVELS)
        q = _expand_to_q(ref_p, ref_q)
        kl = _kl_divergence(hist, q)
        if kl < best:          # (the reference's ternary keeps the OLD bin when kl improves -- an inverted update that
            best, thresh = kl, i   # never mattered there because the threshold is not used; the arg-min is meant)
        start_num += int(hist[i])
    return thresh if thresh > 0 else BIN_NUM


# ------------------------------------------------------------------------------------------------- the calibrator
def fused_chains(graph, optimised_ops):
    """{optimised node: [original nodes it stands for, in order]} -- the head and the single-consumer followers that
    Graph::Optimize merged into it (they are no longer nodes of the optimised graph). optimised_ops: {name: fused op}."""
    nodes = {n["name"]: n for n in graph["nodes"]}
    consumers = {n: [t for t, _ in graph["edges_out"].get(n, [])] for n in nodes}
    chains = {}
    for head, op in optimised_ops.items():
        elt = op == "ConvEltwise"
        allowed = set()
        if "Batchnorm" in op or elt: allowed.add("BatchNorm")
        if "Scale" in op or elt: allowed.add("Scale")
        if "Relu" in op or elt: allowed.add("ReLU")
        if "Pool" in op: allowed.add("Pooling")
        if elt: allowed.add("Eltwise")
        chain, cur = [head], head
        while True:
            outs = consumers.get(cur, [])
            if len(outs) != 1:
                break
            nxt = outs[0]
            if nxt in optimised_ops or nodes[nxt]["op"] not in allowed:
                break
            chain.append(nxt)
            cur = nxt
        chains[head] = chain
    return chains


class Calibrator:
    """Calibrator<NV> over the FP32 net of this library. graph: the anakin_bin graph dict (un-fused, fp32)."""

    def __init__(self, graph, batch_stream, algo="maxabs", device=0):
        assert algo in ("maxabs", "entropy")
        self.graph, self.stream, self.algo, self.device = graph, batch_stream, algo, device
        self.scale_map = {}
        self.max_map = {}
        self.thresh_map = {}

    def _net_for(self, batch):
        G = api.Graph.from_bytes(anakin_bin.dumps(self.graph))
        for n in self.graph["nodes"]:
            if n["op"] == "Input":
                G.ResetBatchSize(n["name"], batch)
        G.Optimize()
        net = api.Net(G, "fp32", device=self.device, calib_stats=True)
        return G, net

    def generate_calibrator_table(self):
        """Two passes (max, histogram), thresholds, scales; returns {node name: scale}."""
        first = next(self.stream.reset())
        batch = int(np.asarray(first).shape[0])
        G, net = self._net_for(batch)
        ops = dict((n, o) for n, o in net.exec_order())
        in_name = net.in_names[0]
        observed = net.calib_names()                       # the input, then every launched op's output
        ops.setdefault(in_name, "Input")

        def run_pass(p):
            net.calib_set_pass(p)
            for x in self.stream.reset():
                x = np.ascontiguousarray(x, np.float32)
                assert x.shape[0] == batch, "calibration batches must share one batch size"
                net.set_input(in_name, x)
                net.prediction()

        net.calib_reset()
        run_pass(0)                                         # pass 1: get_max_values
        maxs, _ = net.calib_read(hist=False)
        maxv = {n: float(maxs[k]) for k, n in enumerate(observed)}
        kl_thresh = {}
        if self.algo == "entropy":
            run_pass(1)                                     # pass 2: get_histgrams (bin width max / BIN_NUM)
            kl_thresh = {n: int(t) for n, t in zip(observed, net.calib_kl())}
        chains = fused_chains(self.graph, ops)
        self.max_map, self.thresh_map, self.scale_map = {}, {}, {}
        for n in observed:
            mx = maxv[n]
            thresh = BIN_NUM
            if self.algo == "entropy" and mx > 0:
                thresh = kl_thresh[n]
            scale = float(np.float32(mx) / np.float32(127 * BIN_NUM) * np.float32(thresh)) if mx > 0 else 1.0
            for member in chains.get(n, [n]):
                self.scale_map[member] = scale
                self.max_map[member] = mx
                self.thresh_map[member] = thresh
        # alias nodes (Split, Flatten, Output) carry the tensor of their producer
        producers = {n["name"]: [b for b, _ in self.graph["edges_in"].get(n["name"], [])] for n in self.graph["nodes"]}
        for n in self.graph["nodes"]:
            nm = n["name"]
            if nm not in self.scale_map and producers[nm] and producers[nm][0] in self.scale_map:
                self.scale_map[nm] = self.scale_map[producers[nm][0]]
                self.max_map[nm] = self.max_map[producers[nm][0]]
        return dict(self.scale_map)

    def write_calibrator(self, path):
        """'<name> <scale>' per line, sorted by name (std::map order) -- entropy_calibrator.cpp:167-177; the scale
        with 9 significant digits (the reference's %f keeps 6 decimals, i.e. 3-4 digits of a typical scale)."""
        with open(path, "w") as f:
            for k in sorted(self.scale_map):
                f.write("%s %.9g\n" % (k, self.scale_map[k]))

    @staticmethod
    def read_calibrator(path):
        table = {}
        with open(path) as f:
            for line in f:
                parts = line.split()
                if len(parts) == 2:
                    table[parts[0]] = float(parts[1])
        return table
