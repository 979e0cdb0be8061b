"""Writes tests/golden/cv2_resize.json: SHA-256 digests of OpenCV's bytes (cv2.resize with INTER_LINEAR, then the
crop; NV12 / I420 frames through cv2.cvtColor first) on the designed cases of tests/cv2_resize_oracle.py, so that the
restatement stays pinned to OpenCV on a machine without it. The bytes are those of OpenCV 4.13 on x86-64.

    python tools/make_cv2_resize_golden.py        (needs cv2)
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cv2_resize_oracle as O  # noqa: E402


def main():
    import cv2
    cases = []
    for i, (h, w, c, s, oh, ow, image) in enumerate(O.GOLDEN_CASES):
        src = O.case_image(h, w, c, image, seed=i)
        out = O.case_resize(src, c, image, s, oh, ow, cv2=True)
        cases.append({"h": h, "w": w, "c": c, "resize_short": s, "out_h": oh, "out_w": ow, "image": image, "seed": i,
                      "sha256": hashlib.sha256(out.tobytes()).hexdigest()})
    doc = {"filter": "cv2_linear", "opencv": cv2.__version__, "platform": "x86-64",
           "image": "case_image(h, w, c, image, seed) of tests/cv2_resize_oracle.py; digest of the uint8 "
                    "[out_h][out_w][c] bytes", "cases": cases}
    path = os.path.join(ROOT, "tests", "golden", "cv2_resize.json")
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("wrote", path, len(cases), "cases")


if __name__ == "__main__":
    main()
