"""Boxes cropped out of one 1920x1080 frame on the GPU (Net.set_input_crops) against the same boxes cut on the host
and sent as images (Net.set_input_images), in one GPU run:
  python tools/bench_image_crops.py [--reps 20]

  - card name, power limit and SM clock (nvidia-smi query, before and after the timings);
  - the ImageResize op's device time (Net.profile_ops with reps > 1), ResNet-50 INT8 at b8 and b32, resize_short 256,
    both filters, k = batch boxes of one frame: crops of an NV12 frame, crops of an RGB frame, and the images path on
    the same boxes cut from the RGB frame on the host; timed in 3 interleaved rounds, median and spread;
  - H2D bytes per request of each form (pixels, sizes and boxes);
  - on one host thread, what a caller without crops does per box: cv2.cvtColor of the NV12 frame (once per frame,
    shown per box), then a Pillow crop with torchvision's Resize + CenterCrop.
Prints one JSON line; writes nothing into the source tree (model files go to a temporary directory)."""
import argparse
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

import crop_oracle as K  # noqa: E402
import yuv_oracle as Y  # noqa: E402

MEAN = [123.675, 116.28, 103.53]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375]
S = 256
FRAME_HW = (1080, 1920)


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
    G.set_input_image_resize("input_0", FRAME_HW[0], FRAME_HW[1], S, filter=filt, pixel_format=pixel_format)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        G = api.Graph.from_file(p)
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return api.Net(G, "int8")


def boxes_of(k, seed):
    """k detector-like boxes of the frame: sides 48..600, anywhere inside it, odd offsets and sizes included."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(k):
        h, w = (int(x) for x in rng.integers(48, 601, 2))
        out.append((0, int(rng.integers(0, FRAME_HW[0] - h + 1)), int(rng.integers(0, FRAME_HW[1] - w + 1)), h, w))
    return out


def op_rows(reps):
    nv12 = Y.random_frame(*FRAME_HW, Y.NV12, seed=1)
    rgb = Y.yuv_to_rgb(nv12, Y.NV12)
    rows = []
    for batch in (8, 32):
        boxes = boxes_of(batch, batch)
        host_crops = [K.crop([rgb], K.INTERLEAVED, b) for b in boxes]
        forms = {   # form: (net format, setter)
            "crops_nv12": ("nv12", lambda n: n.set_input_crops("input_0", [nv12], boxes)),
            "crops_rgb": ("interleaved", lambda n: n.set_input_crops("input_0", [rgb], boxes)),
            "images_rgb": ("interleaved", lambda n: n.set_input_images("input_0", host_crops)),
        }
        h2d = {"crops_nv12": nv12.nbytes + 8 + 20 * batch, "crops_rgb": rgb.nbytes + 8 + 20 * batch,
               "images_rgb": sum(c.nbytes for c in host_crops) + 8 * batch}
        for filt in ("reference", "pil"):
            nets = {f: net_of(batch, filt, f) for f in ("nv12", "interleaved")}
            t = {f: [] for f in forms}
            names = list(forms)
            for f in names:
                fmt, put = forms[f]
                put(nets[fmt])
                nets[fmt].profile_ops(iters=3, reps=1)          # warm-up
            for rnd in range(3):
                for f in names[rnd:] + names[:rnd]:
                    fmt, put = forms[f]
                    put(nets[fmt])
                    prof = nets[fmt].profile_ops(iters=10, reps=reps)
                    assert prof[0][1] == "ImageResize"
                    t[f].append(prof[0][2] * 1e3)
            row = {"model": "resnet50", "precision": "int8", "batch": batch, "filter": filt, "frame_hw": list(FRAME_HW),
                   "resize_short": S, "boxes": boxes}
            for f in names:
                row[f] = {"resize_us": spread(t[f]), "h2d_bytes_per_request": h2d[f]}
            rows.append(row)
            del nets
    return rows


def host_per_box():
    try:
        import cv2
        import torchvision.transforms as T
        from PIL import Image
    except ImportError:
        return None
    cv2.setNumThreads(1)
    nv12 = Y.random_frame(*FRAME_HW, Y.NV12, seed=1)
    boxes = boxes_of(32, 32)
    tf = T.Compose([T.Resize(S, T.InterpolationMode.BILINEAR), T.CenterCrop(224)])
    cvt, per_box = [], []
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in range(10):
            rgb = cv2.cvtColor(nv12, cv2.COLOR_YUV2RGB_NV12)
        cvt.append((time.perf_counter() - t0) / 10 * 1e3)
        im = Image.fromarray(rgb)
        t0 = time.perf_counter()
        for _, t, l, h, w in boxes:
            tf(im.crop((l, t, l + w, t + h)))
        per_box.append((time.perf_counter() - t0) / len(boxes) * 1e3)
    return {"cvtcolor_nv12_ms_per_frame": spread(cvt), "crop_resize_centercrop_ms_per_box": spread(per_box),
            "boxes_per_frame": [8, 32]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs an H100"
    before = card()
    rows = op_rows(a.reps)
    print(json.dumps({"card": before, "card_after": card(), "ops": rows, "host_one_thread": host_per_box()}))


if __name__ == "__main__":
    main()
