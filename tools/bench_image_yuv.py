"""NV12 / I420 frames against interleaved RGB through the on-device resize (the `<input>:ImageResize` op), in one GPU run:
  python tools/bench_image_yuv.py [--reps 20]

  - card name, power limit and SM clock (nvidia-smi query, before and after the timings);
  - the ImageResize op's device time beside the stem op of the same Net (Net.profile_ops with reps > 1), ResNet-50
    INT8 at b8 and b32, resize_short 256, both filters, frames of 1280x720, 1920x1080 and 3840x2160 (w x h): one Net
    per pixel format (interleaved RGB, NV12, I420) with the same weights and the same frames, timed in interleaved
    rounds (3 rounds, the formats in rotating order), median and spread;
  - H2D bytes per request of each format;
  - on one host thread, cv2.cvtColor(frame, COLOR_YUV2RGB_NV12 / _I420) per frame where cv2 is installed: the
    conversion a caller with YUV frames no longer does before handing over RGB.
Prints one JSON line; writes nothing into the source tree (model files go to a temporary directory)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import yuv_oracle as Y  # noqa: E402

MEAN = [123.675, 116.28, 103.53]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375]
S = 256
FRAMES = [(720, 1280), (1080, 1920), (2160, 3840)]      # (h, w)
MAX_HW = (2160, 3840)
FORMATS = ["interleaved", "nv12", "i420"]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    f = [x.strip() for x in r.stdout.strip().split(",")]
    return dict(zip(["name", "power_limit", "sm_clock", "max_sm_clock"], f))


def spread(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}


def net_of(batch, filt, pixel_format):
    from anakin_b200 import anakin_bin, api, modelzoo
    G = api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build("resnet50", batch=batch, precision="int8")))
    G.set_input_image("input_0", MEAN, SCALE, [0, 1, 2])
    G.set_input_image_resize("input_0", MAX_HW[0], MAX_HW[1], S, filter=filt, pixel_format=pixel_format)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        G = api.Graph.from_file(p)
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return api.Net(G, "int8")


def requests(batch, h, w):
    """{format: list of images} of one request: the same frames as NV12, I420 and their RGB."""
    nv12 = [Y.random_frame(h, w, Y.NV12, seed=i) for i in range(batch)]
    i420 = [Y.make_frame(*Y.planes(f, Y.NV12), Y.I420) for f in nv12]
    return {"interleaved": [Y.yuv_to_rgb(f, Y.NV12) for f in nv12], "nv12": nv12, "i420": i420}


def op_rows(reps):
    rows = []
    for batch in (8, 32):
        for filt in ("reference", "pil"):
            nets = {f: net_of(batch, filt, f) for f in FORMATS}
            for h, w in FRAMES:
                req = requests(batch, h, w)
                t = {f: {"resize": [], "stem": []} for f in FORMATS}
                for f in FORMATS:
                    nets[f].set_input_images("input_0", req[f])
                    nets[f].profile_ops(iters=3, reps=1)          # warm-up
                for rnd in range(3):
                    for f in FORMATS[rnd:] + FORMATS[:rnd]:
                        prof = nets[f].profile_ops(iters=10, reps=reps)
                        assert prof[0][1] == "ImageResize"
                        stem = next((n, ms) for n, o, ms in prof if o.startswith("Conv"))
                        t[f]["resize"].append(prof[0][2] * 1e3)
                        t[f]["stem"].append(stem[1] * 1e3)
                row = {"model": "resnet50", "precision": "int8", "batch": batch, "filter": filt, "frame_hw": [h, w],
                       "resize_short": S, "stem_op": stem[0]}
                for f in FORMATS:
                    row[f] = {"resize_us": spread(t[f]["resize"]), "stem_us": spread(t[f]["stem"]),
                              "h2d_bytes_per_request": int(sum(a.nbytes for a in req[f]) + batch * 8)}
                rows.append(row)
            del nets
    return rows


def host_cvtcolor():
    try:
        import cv2
    except ImportError:
        return None
    out = []
    for h, w in FRAMES:
        row = {"frame_hw": [h, w]}
        for name, fmt in (("nv12", Y.NV12), ("i420", Y.I420)):
            frame = Y.random_frame(h, w, fmt, seed=0)
            code = cv2.COLOR_YUV2RGB_NV12 if fmt == Y.NV12 else cv2.COLOR_YUV2RGB_I420
            cv2.setNumThreads(1)
            cv2.cvtColor(frame, code)
            v = []
            for _ in range(3):
                t0 = time.perf_counter()
                for _ in range(20):
                    cv2.cvtColor(frame, code)
                v.append((time.perf_counter() - t0) / 20 * 1e3)
            row[name + "_ms"] = spread(v)
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs an H100"
    before = card()
    rows = op_rows(a.reps)
    print(json.dumps({"card": before, "card_after": card(), "ops": rows, "host_cvtcolor_one_thread": host_cvtcolor()}))


if __name__ == "__main__":
    main()
