"""8-bit image input vs fp32 input, in one GPU run:
  python tools/bench_image_input.py [--reps 20] [--requests 300]

  - card name and power limit (nvidia-smi query);
  - the stem op's device time (Net.profile_ops with reps > 1) for each model built twice, fp32 input and image input:
    ResNet-50 INT8 b8 and b32, MobileNet-v1 FP16 b16, VGG16 FP32 b4; 3 runs in alternating order, median and spread;
  - Worker end-to-end images/s for ResNet-50 INT8 b8, 6 threads, pinned inputs, fp32 vs uint8 requests, with the
    request protocol of bench.py's Worker leg (2 x threads requests in flight);
  - H2D bytes per request, from the shapes;
  - host time of numpy's normalisation (BGR -> RGB, - mean, * scale, HWC -> CHW, fp32) per 224x224 image -- numpy's
    time, not that of a C++ loader.
Prints one JSON line. Writes nothing into the source tree (model files go to a temporary directory)."""
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MEAN = [123.675, 116.28, 103.53]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375]
SRC = [2, 1, 0]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    name, _, power = r.stdout.strip().partition(",")
    return {"name": name.strip(), "power_limit": power.strip()}


def images(batch, seed=1):
    return np.random.default_rng(seed).integers(0, 256, (batch, 224, 224, 3), dtype=np.uint8)


def normalise(u8):
    x = (u8[..., SRC].astype(np.float32) - np.float32(MEAN)) * np.float32(SCALE)
    return np.ascontiguousarray(x.transpose(0, 3, 1, 2))


def blobs(model, precision, batch):
    from anakin_b200 import anakin_bin, api, modelzoo
    blob = anakin_bin.dumps(modelzoo.build(model, batch=batch, precision=precision if precision == "int8" else "fp32"))
    G = api.Graph.from_bytes(blob)
    G.set_input_image("input_0", MEAN, SCALE, SRC)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        with open(p, "rb") as f:
            return blob, f.read()


def net_of(blob, precision, batch):
    from anakin_b200 import api
    G = api.Graph.from_bytes(blob)
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return api.Net(G, precision)


def stem_ms(net, reps):
    for name, op, ms in net.profile_ops(iters=10, reps=reps):
        if op.startswith("Conv"):
            return name, ms
    raise RuntimeError("no convolution in the net")


def spread(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}


def stem_rows(reps):
    rows = []
    for model, precision, batch in [("resnet50", "int8", 8), ("resnet50", "int8", 32), ("mobilenet_v1", "fp16", 16),
                                    ("vgg16", "fp32", 4)]:
        fblob, iblob = blobs(model, precision, batch)
        nf, ni = net_of(fblob, precision, batch), net_of(iblob, precision, batch)
        u8 = images(batch)
        nf.set_input("input_0", normalise(u8))
        ni.set_input_image("input_0", u8)
        t = {"fp32": [], "u8": []}
        for run in range(3):
            order = [("fp32", nf), ("u8", ni)] if run % 2 == 0 else [("u8", ni), ("fp32", nf)]
            for key, net in order:
                name, ms = stem_ms(net, reps)
                t[key].append(ms * 1e3)
        rows.append({"model": model, "precision": precision, "batch": batch, "stem_op": name,
                     "stem_us_fp32": spread(t["fp32"]), "stem_us_u8": spread(t["u8"]),
                     "h2d_bytes_fp32": batch * 3 * 224 * 224 * 4, "h2d_bytes_u8": batch * 224 * 224 * 3})
        del nf, ni
    return rows


def worker_e2e(requests, threads=6, batch=8):
    import torch
    from anakin_b200 import api
    fblob, iblob = blobs("resnet50", "int8", batch)
    u8 = images(batch)
    x = normalise(u8)
    res = {"fp32": [], "u8": []}
    with tempfile.TemporaryDirectory() as d:
        paths = {}
        for key, blob in (("fp32", fblob), ("u8", iblob)):
            paths[key] = os.path.join(d, key + ".anakin.bin")
            with open(paths[key], "wb") as f:
                f.write(blob)
        workers = {k: api.Worker(paths[k], "int8", threads=threads, devices=[0], batch=batch) for k in paths}
        for W in workers.values():
            W.wait_ready()
        depth = 2 * threads
        src = {"fp32": x, "u8": u8}
        bufs = {k: [torch.from_numpy(src[k]).pin_memory() for _ in range(depth)] for k in src}
        outs = [torch.empty(batch * 1000, dtype=torch.float32).pin_memory() for _ in range(depth)]

        def serve(key, n):
            W, inflight = workers[key], 0
            for i in range(n):
                if inflight == depth:
                    W.async_get_result()
                    inflight -= 1
                j = i % depth
                b = bufs[key][j]
                if key == "u8":
                    W.async_prediction_image_ptr(b.data_ptr(), b.numel(), outs[j].data_ptr(), outs[j].numel())
                else:
                    W.async_prediction_ptr(b.data_ptr(), b.numel(), outs[j].data_ptr(), outs[j].numel())
                inflight += 1
            while inflight:
                W.async_get_result()
                inflight -= 1

        for key in ("fp32", "u8"):
            serve(key, max(6 * threads, 100))       # eager run, graph capture, warm replays on every thread
        for run in range(3):
            for key in (("fp32", "u8") if run % 2 == 0 else ("u8", "fp32")):
                t0 = time.perf_counter()
                serve(key, requests)
                res[key].append(batch * requests / (time.perf_counter() - t0))
        del workers
    return {"model": "resnet50", "precision": "int8", "batch": batch, "threads": threads, "requests": requests,
            "images_per_s_fp32": spread(res["fp32"]), "images_per_s_u8": spread(res["u8"]),
            "h2d_bytes_per_request_fp32": x.nbytes, "h2d_bytes_per_request_u8": u8.nbytes}


def numpy_normalise_us(n=64):
    u8 = images(n, seed=2)
    normalise(u8[:4])
    t = []
    for _ in range(5):
        t0 = time.perf_counter()
        normalise(u8)
        t.append((time.perf_counter() - t0) / n * 1e6)
    return {"what": "numpy: BGR->RGB, astype(float32), - mean, * scale, HWC->CHW, per 224x224 image, one host thread",
            "us_per_image": spread(t)}


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--requests", type=int, default=300)
    args = ap.parse_args()
    line = {"card": card(), "stem": stem_rows(args.reps), "worker_e2e": worker_e2e(args.requests),
            "host_normalise": numpy_normalise_us()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
