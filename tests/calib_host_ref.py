"""The host statistics of the calibration tool as they were computed before they moved to the GPU, kept as the yardstick
of the GPU path (tests/test_calibrate_gpu.py, tools/bench_calibrate.py): every edge tensor of a `keep_edges` FP32 net
is read back after prediction() and reduced with numpy -- the max |x| of pass 1, the 2048-bin histogram of |x| of
pass 2 -- and the thresholds come from anakin_b200.calibrate.kl_threshold."""
import concurrent.futures as cf
import multiprocessing as mp
import os

import numpy as np

from anakin_b200 import calibrate

BIN_NUM = calibrate.BIN_NUM


def edge_tensors(net, names, x):
    """(name, fp32 array) of every observed tensor after one prediction on x: the graph input as given, every edge
    without its NHWC channel padding. net: a keep_edges FP32 net; names: the input first."""
    x = np.ascontiguousarray(x, np.float32)
    net.set_input(names[0], x)
    net.prediction()
    net.sync()
    yield names[0], x
    for n in names[1:]:
        arr, info = net.read_tensor(n)
        c = info["dims"][1]
        yield n, (arr[..., :c] if info["layout"] == 9 else arr)


def fold_max(maxv, n, t):
    maxv[n] = max(maxv.get(n, 0.0), float(np.abs(t).max()))


def add_hist(hists, maxv, n, t):
    if maxv[n] <= 0:
        return
    step = np.float32(maxv[n]) / np.float32(BIN_NUM)
    ids = np.minimum((np.abs(t.astype(np.float32)) / step).astype(np.int64), BIN_NUM - 1)
    hists.setdefault(n, np.zeros(BIN_NUM, np.int64))
    hists[n] += np.bincount(ids.ravel(), minlength=BIN_NUM)


def host_stats(net, names, batches, histograms=True):
    """({name: max}, {name: int64 hist}) of the two host passes over `batches`."""
    maxv, hists = {n: 0.0 for n in names}, {}
    for x in batches:
        for n, t in edge_tensors(net, names, x):
            fold_max(maxv, n, t)
    if histograms:
        for x in batches:
            for n, t in edge_tensors(net, names, x):
                add_hist(hists, maxv, n, t)
    return maxv, hists


def kl_at(hist, i):
    """The restatement's KL value of candidate bin i (one iteration of calibrate.kl_threshold)."""
    hist = np.asarray(hist, np.int64)
    total = int(hist.sum() - hist[0])
    start_num = int(hist[1:i].sum())
    ref_p = hist[1:i + 1].copy()
    ref_p[i - 1] += total - start_num
    q = calibrate._expand_to_q(ref_p, calibrate._get_ref_q(ref_p, calibrate.QUANT_LEVELS))
    return calibrate._kl_divergence(hist, q)


def kl_thresholds(hists):
    """calibrate.kl_threshold of every histogram (4 s each in numpy), spread over the host's cores."""
    hists = [np.asarray(h, np.int64) for h in hists]
    workers = max(1, min(len(hists), os.cpu_count() or 1))
    if workers == 1:
        return [calibrate.kl_threshold(h) for h in hists]
    with cf.ProcessPoolExecutor(workers, mp_context=mp.get_context("spawn")) as ex:
        return list(ex.map(calibrate.kl_threshold, hists))


def table_from_stats(graph, ops, names, maxv, thresh):
    """The table assembly of Calibrator.generate_calibrator_table from per-tensor maxima and thresholds: the scale
    formula, fused chains and alias propagation."""
    chains = calibrate.fused_chains(graph, ops)
    scale_map, max_map, thresh_map = {}, {}, {}
    for n in names:
        mx = maxv[n]
        t = thresh.get(n, BIN_NUM) if mx > 0 else BIN_NUM
        scale = float(np.float32(mx) / np.float32(127 * BIN_NUM) * np.float32(t)) if mx > 0 else 1.0
        for member in chains.get(n, [n]):
            scale_map[member], max_map[member], thresh_map[member] = scale, mx, t
    producers = {n["name"]: [b for b, _ in graph["edges_in"].get(n["name"], [])] for n in graph["nodes"]}
    for n in graph["nodes"]:
        nm = n["name"]
        if nm not in scale_map and producers[nm] and producers[nm][0] in scale_map:
            scale_map[nm] = scale_map[producers[nm][0]]
            max_map[nm] = max_map[producers[nm][0]]
    return scale_map, thresh_map
