"""Writes tests/golden/pil_resize.json: SHA-256 digests of Pillow's bytes (torchvision's Resize + CenterCrop for
resize_short > 0, Image.resize(BILINEAR) for a stretch) on the designed cases of tests/pil_resize_oracle.py, so that the
restatement stays pinned to Pillow on a machine without it.

    python tools/make_pil_resize_golden.py        (needs Pillow and torchvision)
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import pil_resize_oracle as P  # noqa: E402


def main():
    import PIL
    import torchvision
    cases = []
    for i, (h, w, c, s, oh, ow, image) in enumerate(P.GOLDEN_CASES):
        img = P.case_image(h, w, c, image, seed=i)
        out = P.pillow_resize(img, s, oh, ow)
        cases.append({"h": h, "w": w, "c": c, "resize_short": s, "out_h": oh, "out_w": ow, "image": image, "seed": i,
                      "sha256": hashlib.sha256(out.tobytes()).hexdigest()})
    doc = {"pillow": PIL.__version__, "torchvision": torchvision.__version__,
           "image": "case_image(h, w, c, image, seed) of tests/pil_resize_oracle.py; digest of the uint8 "
                    "[out_h][out_w][c] bytes", "cases": cases}
    path = os.path.join(ROOT, "tests", "golden", "pil_resize.json")
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("wrote", path, len(cases), "cases")


if __name__ == "__main__":
    main()
