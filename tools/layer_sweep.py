"""Device-bound sweep of the conv kernel variants over the distinct ResNet-50 layer shapes (INT8).

Every (layer, variant) is timed as a CUDA graph of `--chain` back-to-back launches of ONE plan on the capture stream
(programmatic dependent launch between them, exactly as Net::prediction() replays them), so the host cost of a C-ABI
call (~7 us through ctypes) is out of the number. Variants: tile width (B200_SABER_FORCE_BN), kernel family
(B200_SABER_SLAB / B200_SABER_PERSISTENT), split-K factor (B200_SABER_FORCE_SPLIT); `auto` is what the planner picks.
  python tools/layer_sweep.py [--batch 8] [--chain 20] [--full]
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from anakin_b200 import saber_abi as A  # noqa: E402
from gpu_util import ConvRunner, dev  # noqa: E402

# name, h, c, k, r, stride, pad, residual, relu, count in ResNet-50
LAYERS = [
    ("s2a br1 1x1 64>256", 56, 64, 256, 1, 1, 0, False, False, 1),
    ("s2a 2a 1x1 64>64", 56, 64, 64, 1, 1, 0, False, True, 1),
    ("s2 2b 3x3 64", 56, 64, 64, 3, 1, 1, False, True, 3),
    ("s2 2c 1x1 64>256 +res", 56, 64, 256, 1, 1, 0, True, True, 3),
    ("s2 2a 1x1 256>64", 56, 256, 64, 1, 1, 0, False, True, 2),
    ("s3a br1 1x1/2 256>512", 56, 256, 512, 1, 2, 0, False, False, 1),
    ("s3a 2a 1x1/2 256>128", 56, 256, 128, 1, 2, 0, False, True, 1),
    ("s3 2b 3x3 128", 28, 128, 128, 3, 1, 1, False, True, 4),
    ("s3 2c 1x1 128>512 +res", 28, 128, 512, 1, 1, 0, True, True, 4),
    ("s3 2a 1x1 512>128", 28, 512, 128, 1, 1, 0, False, True, 3),
    ("s4a br1 1x1/2 512>1024", 28, 512, 1024, 1, 2, 0, False, False, 1),
    ("s4a 2a 1x1/2 512>256", 28, 512, 256, 1, 2, 0, False, True, 1),
    ("s4 2b 3x3 256", 14, 256, 256, 3, 1, 1, False, True, 6),
    ("s4 2c 1x1 256>1024 +res", 14, 256, 1024, 1, 1, 0, True, True, 6),
    ("s4 2a 1x1 1024>256", 14, 1024, 256, 1, 1, 0, False, True, 5),
    ("s5a br1 1x1/2 1024>2048", 14, 1024, 2048, 1, 2, 0, False, False, 1),
    ("s5a 2a 1x1/2 1024>512", 14, 1024, 512, 1, 2, 0, False, True, 1),
    ("s5 2b 3x3 512", 7, 512, 512, 3, 1, 1, False, True, 3),
    ("s5 2c 1x1 512>2048 +res", 7, 512, 2048, 1, 1, 0, True, True, 3),
    ("s5 2a 1x1 2048>512", 7, 2048, 512, 1, 1, 0, False, True, 2),
]
ENV_KEYS = ("B200_SABER_PERSISTENT", "B200_SABER_SLAB", "B200_SABER_FORCE_BN", "B200_SABER_FORCE_SPLIT")


def variants(r, full):
    v = [("auto", {})]
    for bn in (32, 64, 128, 256):
        v.append(("tile/%d" % bn, {"B200_SABER_FORCE_BN": str(bn), "B200_SABER_SLAB": "0", "B200_SABER_PERSISTENT": "0"}))
    if r > 1:
        for bn in (32, 64, 128):
            v.append(("slab/%d" % bn, {"B200_SABER_FORCE_BN": str(bn), "B200_SABER_SLAB": "2", "B200_SABER_PERSISTENT": "0"}))
    if full:
        for bn in (32, 64, 128, 256):
            v.append(("pers/%d" % bn, {"B200_SABER_FORCE_BN": str(bn), "B200_SABER_SLAB": "0", "B200_SABER_PERSISTENT": "2"}))
        for bn, splits in ((32, (2, 4)), (64, (2, 4)), (128, (2, 4, 8))):
            for sp in splits:
                v.append(("split%d/%d" % (sp, bn), {"B200_SABER_FORCE_BN": str(bn), "B200_SABER_SLAB": "0",
                                                    "B200_SABER_PERSISTENT": "0", "B200_SABER_FORCE_SPLIT": str(sp)}))
    return v


def time_plan(n, h, c, k, r, stride, pad, with_res, relu, env, chain):
    for key in ENV_KEYS:
        os.environ.pop(key, None)
    os.environ.update(env)
    rng = np.random.default_rng(0)
    x = rng.integers(0, 256, (n, h, h, c)).astype(np.uint8)
    wt = rng.integers(-127, 128, (k, c, r, r)).astype(np.int8)
    run = ConvRunner(A.MATH_I8, x.shape, A.UINT8, wt, np.zeros(k, np.float32), np.full(k, 1e-4, np.float32),
                     A.UINT8 if relu else A.INT8, res_dtype=(A.UINT8 if with_res else -1), stride=(stride, stride),
                     pad=(pad, pad), relu=relu)
    info = run.info()
    xd = dev(x)
    res = dev(rng.integers(0, 256, (n, run.ho, run.wo, k)).astype(np.uint8)) if with_res else None
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        out = run.run(xd, res)
        for _ in range(3):
            run.run(xd, res, out_dev=out)
        side.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            for _ in range(chain):
                run.run(xd, res, out_dev=out)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = 1e9
    for _ in range(3):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) / chain * 1e3)
    tag = "slab" if info["slab"] else ("pers" if info["persistent"] else "tile")
    what = "%s/%d/%dx%d" % (tag, info["block_n"], info["grid_x"], info["grid_y"]) + ("/s%d" % info["split"] if info["split"] > 1 else "")
    return best, what


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--chain", type=int, default=20)
    ap.add_argument("--full", action="store_true")
    a = ap.parse_args()
    print("batch %d, INT8 u8 in / u8 out; us per launch inside a %d-launch PDL chain (CUDA graph replay)" % (a.batch, a.chain))
    tot_auto = tot_best = 0.0
    for name, h, c, k, r, stride, pad, wr, relu, count in LAYERS:
        cells, seen = [], {}
        for vname, env in variants(r, a.full):
            try:
                us, what = time_plan(a.batch, h, c, k, r, stride, pad, wr, relu, env, a.chain)
            except Exception as e:   # a variant that does not apply
                continue
            if what in seen and vname != "auto":
                continue
            seen[what] = us
            cells.append((us, vname, what))
        auto = [c_ for c_ in cells if c_[1] == "auto"][0]
        best = min(cells)
        tot_auto += auto[0] * count
        tot_best += best[0] * count
        print("%-26s x%d auto %6.2f %-18s best %6.2f %-18s | " % (name, count, auto[0], auto[2], best[0], best[2]) +
              " ".join("%s=%.2f" % (w, u) for u, _, w in sorted(cells, key=lambda t: t[2])))
        sys.stdout.flush()
    print("sum over the 52 non-stem conv layers: auto %.1f us, best-of-sweep %.1f us" % (tot_auto, tot_best))


if __name__ == "__main__":
    main()
