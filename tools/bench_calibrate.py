"""Wall time of INT8 calibration on the GPU path (Net(calib_stats=True): b200_calib_stats_run inside the captured
prediction, b200_calib_kl_run over all histograms) against the host restatement it replaced (edge read-back + numpy +
calibrate.kl_threshold in Python, tests/calib_host_ref.py).

For every model, batch size and algo, on N synthetic images (N rounded down to whole batches), one JSON line:
  device_s     pass 1 (maxima), pass 2 (histograms; entropy only) and the KL search, each ended by a stream sync
  host_s       the host restatement, timed on a bounded subset (--host-batches batches, --host-kl histograms) and
               scaled to the whole run ("projected"): read-back + numpy per batch and pass, Python KL per tensor
  equal        on that subset: maxima bit for bit, histograms as integer arrays, and the thresholds of the --host-kl
               histograms (a differing threshold is reported with the restatement's KL at both bins)
  gpu          the card's name and power limit, read in the same run

  python tools/bench_calibrate.py [--models resnet50,resnet101] [--images 1000] [--batches 8,32]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from anakin_b200 import anakin_bin, api, calibrate, modelzoo  # noqa: E402
import calib_host_ref as H  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the numbers are unlabelled without it, so say so
        return {"name": "unknown", "power_limit": "unknown (%s)" % e}


def graph(name, batch):
    g = modelzoo.build(name, batch=batch)
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return g, G


def device_run(net, xs, entropy):
    t = {}
    net.calib_reset()
    for p in ((0, 1) if entropy else (0,)):
        net.calib_set_pass(p)
        t0 = time.perf_counter()
        for x in xs:
            net.set_input("input_0", x)
            net.prediction()
        net.sync()
        t["pass%d" % (p + 1)] = time.perf_counter() - t0
    mx, hs = net.calib_read(hist=entropy)
    th = None
    if entropy:
        t0 = time.perf_counter()
        th = net.calib_kl()
        t["kl"] = time.perf_counter() - t0
    return t, mx, hs, th


def bench(name, batch, images, host_batches, host_kl, algo):
    entropy = algo == "entropy"
    nb = max(1, images // batch)
    xs = [modelzoo.synthetic_input(batch, 224, seed=5000 + batch * b) for b in range(min(nb, 4))]
    xs = [xs[b % len(xs)] for b in range(nb)]          # N images from a few distinct batches (host memory)
    _, G = graph(name, batch)
    net = api.Net(G, "fp32", calib_stats=True)
    names = net.calib_names()
    device_run(net, xs[:1], entropy)                     # warm-up: plans, CUDA graph capture
    t_dev, _, _, _ = device_run(net, xs, entropy)
    # the same statistics on the host subset, both ways
    sub = xs[:host_batches]
    _, mx, hs, th = device_run(net, sub, entropy)
    del net
    twin = api.Net(G, "fp32", keep_edges=True)
    t0 = time.perf_counter()
    hmax, _ = H.host_stats(twin, names, sub, histograms=False)
    t_host_p1 = (time.perf_counter() - t0) / len(sub)
    res = {"model": name, "batch": batch, "images": nb * batch, "algo": algo, "tensors": len(names),
           "device_s": {k: round(v, 4) for k, v in t_dev.items()}}
    res["device_s"]["total"] = round(sum(t_dev.values()), 4)
    equal = {"max_bits": all(np.float32(hmax[n]).view(np.uint32) == mx[k].view(np.uint32)
                             for k, n in enumerate(names))}
    host = {"pass1_per_batch": round(t_host_p1, 4), "pass1_projected": round(t_host_p1 * nb, 2)}
    if entropy:
        t0 = time.perf_counter()
        hists = {}
        for x in sub:
            for n, t in H.edge_tensors(twin, names, x):
                H.add_hist(hists, hmax, n, t)
        t_host_p2 = (time.perf_counter() - t0) / len(sub)
        equal["hist"] = all((hs[k].astype(np.int64) == hists.get(n, np.zeros(H.BIN_NUM, np.int64))).all()
                            for k, n in enumerate(names))
        live = [k for k, n in enumerate(names) if hmax[n] > 0][:host_kl]
        t0 = time.perf_counter()
        ref = [calibrate.kl_threshold(hists[names[k]]) for k in live]
        t_kl = (time.perf_counter() - t0) / max(1, len(live))
        diff = [{"tensor": names[k], "gpu": int(th[k]), "host": r, "kl_gpu_bin": H.kl_at(hists[names[k]], int(th[k])),
                 "kl_host_bin": H.kl_at(hists[names[k]], r)} for k, r in zip(live, ref) if int(th[k]) != r]
        equal["thresholds_checked"] = len(live)
        equal["thresholds_differing"] = diff
        host.update({"pass2_per_batch": round(t_host_p2, 4), "pass2_projected": round(t_host_p2 * nb, 2),
                     "kl_per_tensor": round(t_kl, 3), "kl_projected": round(t_kl * len(names), 1)})
    host["total_projected"] = round(sum(v for k, v in host.items() if k.endswith("projected")), 1)
    res["host_s"] = host
    res["host_subset"] = {"batches": len(sub), "kl_tensors": host_kl if entropy else 0}
    res["equal"] = equal
    res["speedup_projected"] = round(host["total_projected"] / res["device_s"]["total"], 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="resnet50")
    ap.add_argument("--images", type=int, default=1000)
    ap.add_argument("--batches", default="8,32")
    ap.add_argument("--algos", default="maxabs,entropy")
    ap.add_argument("--host-batches", type=int, default=2)
    ap.add_argument("--host-kl", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    for m in a.models.split(","):
        for b in [int(v) for v in a.batches.split(",")]:
            for algo in a.algos.split(","):
                r = bench(m, b, a.images, a.host_batches, a.host_kl, algo)
                r["gpu"] = info
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
