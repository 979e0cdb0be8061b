"""Writes tests/golden/yuv_resize.json: SHA-256 digests of OpenCV's cvtColor(COLOR_YUV2RGB_NV12 / _I420) on the
exhaustive frame of tests/yuv_oracle.py (every (Y, U, V) triple), and of cvtColor followed by Pillow's bytes
(torchvision's Resize + CenterCrop for resize_short > 0, Image.resize(BILINEAR) for a stretch) on its designed frames,
so that the restatement stays pinned to OpenCV and Pillow on a machine without them.

    python tools/make_yuv_golden.py        (needs cv2, Pillow and torchvision)
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import pil_resize_oracle as P  # noqa: E402
import yuv_oracle as Y  # noqa: E402


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def main():
    import cv2
    import PIL
    import torchvision
    exhaustive = {name: sha(Y.cv2_rgb(Y.exhaustive_frame(fmt), fmt)) for name, fmt in Y.FORMATS.items()}
    cases = []
    for i, (h, w, s, oh, ow) in enumerate(Y.GOLDEN_CASES):
        for name, fmt in Y.FORMATS.items():
            frame = Y.golden_frame(h, w, fmt, i)
            out = P.pillow_resize(Y.cv2_rgb(frame, fmt), s, oh, ow)
            cases.append({"format": name, "h": h, "w": w, "resize_short": s, "out_h": oh, "out_w": ow, "index": i,
                          "sha256": sha(out)})
    doc = {"cv2": cv2.__version__, "pillow": PIL.__version__, "torchvision": torchvision.__version__,
           "exhaustive": exhaustive,
           "image": "exhaustive: cvtColor of exhaustive_frame(format), uint8 [4096][4096][3]; cases: the uint8 "
                    "[out_h][out_w][3] bytes of the Pillow resize of cvtColor(golden_frame(h, w, format, index)), "
                    "tests/yuv_oracle.py",
           "cases": cases}
    path = os.path.join(ROOT, "tests", "golden", "yuv_resize.json")
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("wrote", path, len(cases), "cases")


if __name__ == "__main__":
    main()
