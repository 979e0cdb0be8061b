"""Writes tests/golden/pil_resize.json and tests/golden/pil_bicubic_resize.json: SHA-256 digests of Pillow's bytes
(torchvision's Resize + CenterCrop for resize_short > 0, Image.resize for a stretch) with the BILINEAR filter on the
designed cases of tests/pil_resize_oracle.py and the BICUBIC filter on those of tests/pil_bicubic_oracle.py, so that
the restatements stay pinned to Pillow on a machine without it. The bicubic bytes are those of x86-64 Pillow, which
evaluates the filter without contraction into fused multiply-adds; a build that contracts can round a weight
differently.

    python tools/make_pil_resize_golden.py        (needs Pillow and torchvision)
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import pil_bicubic_oracle as B  # noqa: E402
import pil_resize_oracle as P  # noqa: E402


def write(name, oracle, head):
    import PIL
    import torchvision
    cases = []
    for i, (h, w, c, s, oh, ow, image) in enumerate(oracle.GOLDEN_CASES):
        img = oracle.case_image(h, w, c, image, seed=i)
        out = oracle.pillow_resize(img, s, oh, ow)
        cases.append({"h": h, "w": w, "c": c, "resize_short": s, "out_h": oh, "out_w": ow, "image": image, "seed": i,
                      "sha256": hashlib.sha256(out.tobytes()).hexdigest()})
    doc = dict(head)
    doc.update({"pillow": PIL.__version__, "torchvision": torchvision.__version__,
                "image": "case_image(h, w, c, image, seed) of tests/%s.py; digest of the uint8 [out_h][out_w][c] "
                         "bytes" % oracle.__name__, "cases": cases})
    path = os.path.join(ROOT, "tests", "golden", name)
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("wrote", path, len(cases), "cases")


def main():
    write("pil_resize.json", P, {})
    write("pil_bicubic_resize.json", B, {"filter": "bicubic", "platform": "x86-64 (no fused multiply-add in the filter)"})


if __name__ == "__main__":
    main()
