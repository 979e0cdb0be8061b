"""Server-side batching in the Worker: ResNet-50 INT8 served to closed-loop clients that each send 1-image requests.

Arms (each with the same --workers Worker threads on one GPU and the same --clients client threads):
  b1            batch-1 Workers without batching: every image is one whole prediction (the baseline)
  b8/dNNN       a batching Worker built at batch 8, max_delay_us NNN for each of --delays
  b32/dNNN      the same at batch 32
Every client keeps one request in flight: it queues a 1-image view request on its own pinned input and output buffers
(Worker.async_prediction_ptr, zero-copy) and waits for it before sending the next. The Worker returns async results in
submission order, so one collector thread calls async_get_result in that order and stamps each request's completion.
One JSON line per arm:
  img_s              completed images / wall time of the timed window
  p50_ms, p99_ms     request latency, host clock from submit to result
  images_per_batch   mean images per executed prediction (Worker.batch_stats; 1 for b1)
and first a line with the card's name, power limit and maximum SM clock, read in the same run.

  python tools/bench_batching.py [--delays 0,200,1000] [--clients 16] [--workers 2] [--seconds 5]
"""
import argparse
import json
import os
import queue
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from anakin_b200 import api, modelzoo  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers are unlabelled without it, so say so
        return {"name": "unknown", "power_limit": "unknown (%s)" % e}


def run_arm(path, batch, delay, clients, workers, seconds, warmup):
    import torch
    w = api.Worker(path, "int8", threads=workers, devices=(0,), batch=batch, max_delay_us=delay)
    w.wait_ready()
    per_in = 3 * 224 * 224
    out_n = w.output_count() // batch
    xs = modelzoo.synthetic_input(clients, 224, seed=77)
    ins = [torch.from_numpy(xs[c].reshape(-1).copy()).pin_memory() for c in range(clients)]
    outs = [torch.zeros(out_n, dtype=torch.float32).pin_memory() for _ in range(clients)]
    submit_lock = threading.Lock()
    inflight = queue.Queue()         # (client, submit time) in the Worker's submission order
    done = [threading.Event() for _ in range(clients)]
    lat = [[] for _ in range(clients)]
    state = {"stop": False, "t0": None, "t1": None}

    def collector():
        while True:
            item = inflight.get()
            if item is None:
                return
            c, t_sub = item
            w.async_get_result()
            t = time.perf_counter()
            t0, t1 = state["t0"], state["t1"]
            if t0 is not None and t_sub >= t0 and (t1 is None or t <= t1):
                lat[c].append(t - t_sub)
            done[c].set()

    def client(c):
        while not state["stop"]:
            done[c].clear()
            with submit_lock:
                t_sub = time.perf_counter()
                w.async_prediction_ptr(ins[c].data_ptr(), per_in, outs[c].data_ptr(), out_n)
                inflight.put((c, t_sub))
            done[c].wait()

    col = threading.Thread(target=collector)
    col.start()
    ths = [threading.Thread(target=client, args=(c,)) for c in range(clients)]
    for t in ths:
        t.start()
    time.sleep(warmup)
    stats0 = w.batch_stats() if delay is not None else None
    state["t0"] = time.perf_counter()
    time.sleep(seconds)
    state["t1"] = time.perf_counter()
    stats1 = w.batch_stats() if delay is not None else None
    state["stop"] = True
    for t in ths:
        t.join()
    inflight.put(None)
    col.join()
    del w
    all_lat = np.array([x for l in lat for x in l]) * 1e3
    wall = state["t1"] - state["t0"]
    fill = 1.0 if stats0 is None else (stats1[1] - stats0[1]) / max(1, stats1[0] - stats0[0])
    return {"img_s": round(len(all_lat) / wall, 1), "p50_ms": round(float(np.percentile(all_lat, 50)), 3),
            "p99_ms": round(float(np.percentile(all_lat, 99)), 3), "images_per_batch": round(fill, 2),
            "requests": int(len(all_lat))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--delays", default="0,200,1000")
    ap.add_argument("--batches", default="8,32")
    ap.add_argument("--clients", type=int, default=16)
    ap.add_argument("--workers", type=int, default=2)
    ap.add_argument("--seconds", type=float, default=5.0)
    ap.add_argument("--warmup", type=float, default=2.0)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info(), "model": "resnet50", "precision": "int8", "clients": args.clients,
                      "workers": args.workers}), flush=True)
    with tempfile.TemporaryDirectory() as d:
        paths = {}
        for b in [1] + [int(x) for x in args.batches.split(",")]:
            paths[b] = os.path.join(d, "resnet50_b%d.anakin.bin" % b)
            modelzoo.save(modelzoo.build("resnet50", batch=b, precision="int8"), paths[b])
        arms = [("b1", 1, None)] + [("b%d/d%d" % (b, dl), b, dl) for b in [int(x) for x in args.batches.split(",")]
                                    for dl in [int(x) for x in args.delays.split(",")]]
        for name, b, dl in arms:
            r = run_arm(paths[b], b, dl, args.clients, args.workers, args.seconds, args.warmup)
            print(json.dumps(dict(arm=name, batch=b, max_delay_us=dl, **r)), flush=True)


if __name__ == "__main__":
    main()
