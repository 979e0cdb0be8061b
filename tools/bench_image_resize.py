"""On-device resize + centre crop of 8-bit images (the `<input>:ImageResize` op), in one GPU run:
  python tools/bench_image_resize.py [--reps 20] [--requests 300]

  - card name and power limit (nvidia-smi query);
  - the ImageResize op's device time beside the stem op of the same Net (Net.profile_ops with reps > 1), ResNet-50
    INT8 b8 and b32, sources 500x375, 640x480 and 1280x960 (w x h) at resize_short 256; algorithmic bytes (every source
    byte read once plus n*224*224*3 written) and that over the op's time, against the 3.35 TB/s of the H100 SXM data
    sheet. The kernel reads only the 2 x 2 taps of each output pixel, so on a large downscale it touches fewer source
    bytes than the algorithmic count;
  - Worker end-to-end images/s, ResNet-50 INT8 b8, 6 threads, pinned requests (bench.py's Worker protocol, 2 x threads
    in flight): pre-resized 224x224 requests to the plain image Net vs raw 500x375 requests resized on the GPU;
  - H2D bytes per request;
  - OpenCV resize (INTER_LINEAR) + centre crop per image on one host thread, where cv2 is installed.
  Every timing is 3 runs in alternating order, median and spread. Prints one JSON line; writes nothing into the source
  tree (model files go to a temporary directory)."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

MEAN = [123.675, 116.28, 103.53]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375]
SRC = [2, 1, 0]
S = 256
HBM_TBS = 3.35
SOURCES = [(375, 500), (480, 640), (960, 1280)]      # (h, w)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    name, _, power = r.stdout.strip().partition(",")
    return {"name": name.strip(), "power_limit": power.strip()}


def spread(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}


def images(n, h, w, seed=1):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(n)]


def model_blob(batch, max_hw=None):
    """The ResNet-50 INT8 model with an image input, resizing (max_hw given) or fixed-size."""
    from anakin_b200 import anakin_bin, api, modelzoo
    G = api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build("resnet50", batch=batch, precision="int8")))
    G.set_input_image("input_0", MEAN, SCALE, SRC)
    if max_hw:
        G.set_input_image_resize("input_0", max_hw[0], max_hw[1], S)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        with open(p, "rb") as f:
            return f.read()


def net_of(blob, batch):
    from anakin_b200 import api
    G = api.Graph.from_bytes(blob)
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return api.Net(G, "int8")


def op_rows(reps):
    rows = []
    for batch in (8, 32):
        net = net_of(model_blob(batch, max_hw=(960, 1280)), batch)
        for h, w in SOURCES:
            net.set_input_images("input_0", images(batch, h, w))
            t = {"resize": [], "stem": []}
            for _ in range(3):
                prof = net.profile_ops(iters=10, reps=reps)
                assert prof[0][1] == "ImageResize"
                stem = next((n, ms) for n, o, ms in prof if o.startswith("Conv"))
                t["resize"].append(prof[0][2] * 1e3)
                t["stem"].append(stem[1] * 1e3)
            nbytes = batch * (h * w * 3 + 224 * 224 * 3)
            med = statistics.median(t["resize"])
            rows.append({"model": "resnet50", "precision": "int8", "batch": batch, "source_hw": [h, w],
                         "resize_short": S, "resize_us": spread(t["resize"]), "stem_op": stem[0],
                         "stem_us": spread(t["stem"]), "algorithmic_bytes": nbytes,
                         "algorithmic_GBps": nbytes / med / 1e3, "share_of_hbm_datasheet": nbytes / med / 1e6 / HBM_TBS})
        del net
    return rows


def worker_e2e(requests, threads=6, batch=8):
    import torch
    from anakin_b200 import api
    h, w = SOURCES[0]
    raw = images(batch, h, w, seed=3)
    import image_resize_oracle as O
    pre = O.resize_batch(raw, S, 224, 224)
    pix, hw = api.pack_images(raw)
    res = {"pre_resized": [], "gpu_resize": []}
    with tempfile.TemporaryDirectory() as d:
        paths = {"pre_resized": os.path.join(d, "fixed.anakin.bin"), "gpu_resize": os.path.join(d, "resize.anakin.bin")}
        for key, blob in (("pre_resized", model_blob(batch)), ("gpu_resize", model_blob(batch, max_hw=(h, w)))):
            with open(paths[key], "wb") as f:
                f.write(blob)
        workers = {k: api.Worker(paths[k], "int8", threads=threads, devices=[0], batch=batch) for k in paths}
        for W in workers.values():
            W.wait_ready()
        depth = 2 * threads
        fixed = [torch.from_numpy(pre).pin_memory() for _ in range(depth)]
        pixs = [(torch.from_numpy(pix).pin_memory(), torch.from_numpy(hw).pin_memory()) for _ in range(depth)]
        outs = [torch.empty(batch * 1000, dtype=torch.float32).pin_memory() for _ in range(depth)]

        def serve(key, n):
            W, inflight = workers[key], 0
            for i in range(n):
                if inflight == depth:
                    W.async_get_result()
                    inflight -= 1
                j = i % depth
                if key == "pre_resized":
                    b = fixed[j]
                    W.async_prediction_image_ptr(b.data_ptr(), b.numel(), outs[j].data_ptr(), outs[j].numel())
                else:
                    p, q = pixs[j]
                    W.async_prediction_images_ptr(p.data_ptr(), p.numel(), q.data_ptr(), batch, outs[j].data_ptr(),
                                                  outs[j].numel())
                inflight += 1
            while inflight:
                W.async_get_result()
                inflight -= 1

        for key in res:
            serve(key, max(6 * threads, 100))       # eager run, graph capture, warm replays on every thread
        for run in range(3):
            for key in (("pre_resized", "gpu_resize") if run % 2 == 0 else ("gpu_resize", "pre_resized")):
                t0 = time.perf_counter()
                serve(key, requests)
                res[key].append(batch * requests / (time.perf_counter() - t0))
        del workers
    return {"model": "resnet50", "precision": "int8", "batch": batch, "threads": threads, "requests": requests,
            "source_hw": [h, w], "images_per_s_pre_resized": spread(res["pre_resized"]),
            "images_per_s_gpu_resize": spread(res["gpu_resize"]),
            "h2d_bytes_per_request_pre_resized": pre.nbytes,
            "h2d_bytes_per_request_gpu_resize": pix.nbytes + hw.nbytes + batch * 32}


def host_cv2_us(n=64):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    import image_resize_oracle as O
    out = {}
    for h, w in SOURCES:
        imgs = images(n, h, w, seed=4)
        rh, rw, top, left = O.geometry(h, w, S, 224, 224)
        t = []
        for _ in range(3):
            t0 = time.perf_counter()
            for a in imgs:
                np.ascontiguousarray(cv2.resize(a, (rw, rh), interpolation=cv2.INTER_LINEAR)[top:top + 224, left:left + 224])
            t.append((time.perf_counter() - t0) / n * 1e6)
        out["%dx%d" % (w, h)] = spread(t)
    return {"what": "cv2.resize INTER_LINEAR + 224 centre crop per image, one host thread", "us_per_image": out}


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--requests", type=int, default=300)
    args = ap.parse_args()
    line = {"card": card(), "ops": op_rows(args.reps), "worker_e2e": worker_e2e(args.requests),
            "host_cv2": host_cv2_us()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
