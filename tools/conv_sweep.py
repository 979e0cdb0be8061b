"""Throughput of the wgmma implicit-GEMM conv kernel alone over a size sweep (CUDA events around
back-to-back launches through the C ABI): TOP/s, fraction of the measured tensor roof and of the
HBM roof for the algorithmic bytes.  python tools/conv_sweep.py [i8|f16|tf32x3]"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from anakin_b200 import saber_abi as A  # noqa: E402
from gpu_util import ConvRunner, dev  # noqa: E402

# n, h, w, c, k, r, stride, pad
SHAPES = [
    (8, 56, 56, 64, 256, 1, 1, 0), (8, 56, 56, 64, 64, 3, 1, 1), (8, 28, 28, 128, 128, 3, 1, 1),
    (8, 14, 14, 256, 256, 3, 1, 1), (8, 7, 7, 512, 512, 3, 1, 1), (8, 14, 14, 1024, 256, 1, 1, 0),
    (32, 56, 56, 64, 256, 1, 1, 0), (32, 28, 28, 128, 128, 3, 1, 1), (32, 14, 14, 256, 256, 3, 1, 1),
    (128, 28, 28, 128, 128, 3, 1, 1), (128, 14, 14, 256, 256, 3, 1, 1), (64, 56, 56, 256, 256, 3, 1, 1),
    (256, 14, 14, 1024, 1024, 1, 1, 0), (64, 28, 28, 512, 512, 3, 1, 1),
]


def main(kind="i8"):
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(
        os.path.join(ROOT, "MEASURED_PEAKS.json")) else {"bf16_tflops": 1590.0, "hbm_gbs": 6650.0}
    mult = {"i8": 2.0, "f16": 1.0, "tf32x3": 0.5 / 3}[kind]
    roof = peaks["bf16_tflops"] * mult
    print("kind %s  tensor roof %.0f T(FL)OP/s (measured bf16 x%.2f)  HBM %.0f GB/s" % (kind, roof, mult, peaks["hbm_gbs"]))
    print("%-34s %5s %9s %9s %8s %8s" % ("n,h,w,c,k,r,s,p", "BN", "us", "TOP/s", "%tensor", "%hbm"))
    rng = np.random.default_rng(0)
    for (n, h, w, c, k, r, stride, pad) in SHAPES:
        if kind == "i8":
            x = rng.integers(-128, 128, (n, h, w, c)).astype(np.int8)
            wt = rng.integers(-127, 128, (k, c, r, r)).astype(np.int8)
            run = ConvRunner(A.MATH_I8, x.shape, A.INT8, wt, np.zeros(k, np.float32), np.full(k, 1e-4, np.float32),
                             A.UINT8, stride=(stride, stride), pad=(pad, pad), relu=True)
            es_in, es_out = 1, 1
        else:
            dt, math, tdt = {"f16": (np.float16, A.MATH_F16, A.HALF), "tf32x3": (np.float32, A.MATH_TF32X3, A.FLOAT)}[kind]
            x = rng.uniform(-1, 1, (n, h, w, c)).astype(dt)
            wt = rng.uniform(-1, 1, (k, c, r, r)).astype(dt)
            run = ConvRunner(math, x.shape, tdt, wt, np.zeros(k, np.float32), None, tdt, stride=(stride, stride),
                             pad=(pad, pad), relu=True)
            es_in = es_out = np.dtype(dt).itemsize
        xd = dev(x)
        out = run.run(xd)
        for _ in range(5):
            run.run(xd, out_dev=out)
        torch.cuda.synchronize()
        reps = 50
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            run.run(xd, out_dev=out)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / reps * 1e3
        M = n * run.ho * run.wo
        ops = 2.0 * M * k * c * r * r
        byts = x.size * es_in + M * k * es_out + wt.size * es_in
        tops = ops / us / 1e6
        print("%-34s %5d %9.2f %9.1f %7.1f%% %7.1f%%" % ("%d,%d,%d,%d,%d,%d,%d,%d" % (n, h, w, c, k, r, stride, pad),
                                                          run.info()["block_n"], us, tops, 100 * tops / roof,
                                                          100 * byts / us / 1e3 / peaks["hbm_gbs"]))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "i8")
