"""Micro-benchmark of single C-ABI kernels (CUDA events around a back-to-back loop).
  python tools/bench_op.py            # pooling / softmax shapes of ResNet-50 at batch 8
"""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from anakin_b200 import saber_abi as A  # noqa: E402
from gpu_util import dev, ptr, stream_ptr  # noqa: E402


def timeit(fn, reps=200):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def pool(n, h, w, c, win, stride, ptype, glob, dtype=A.UINT8):
    lib = A.load()
    d = A.PoolDesc()
    d.dtype, d.type, d.n, d.h, d.w, d.c = dtype, ptype, n, h, w, c
    d.window_h = d.window_w = win
    d.stride_h = d.stride_w = stride
    d.global_pooling = int(glob)
    oh, ow = C.c_int32(), C.c_int32()
    lib.b200_pool_out_hw(C.byref(d), C.byref(oh), C.byref(ow))
    x = dev(np.random.default_rng(0).integers(0, 255, (n, h, w, c)).astype(np.uint8))
    out = torch.zeros((n, oh.value, ow.value, c), dtype=torch.uint8, device="cuda")
    return lambda: lib.b200_pool_run(C.byref(d), ptr(x), ptr(out), stream_ptr())


def softmax(rows, n):
    lib = A.load()
    x = dev(np.random.default_rng(0).uniform(-5, 5, (rows, n)).astype(np.float32))
    out = torch.empty_like(x)
    return lambda: lib.b200_softmax_run(ptr(x), ptr(out), rows, n, 1, stream_ptr())


if __name__ == "__main__":
    for name, fn in [("pool1 8x112x112x64 3x3/2 max", pool(8, 112, 112, 64, 3, 2, 1, False)),
                     ("pool5 8x7x7x2048 global avg", pool(8, 7, 7, 2048, 7, 1, 2, True)),
                     ("pool5 32x7x7x2048 global avg", pool(32, 7, 7, 2048, 7, 1, 2, True)),
                     ("softmax 8x1000", softmax(8, 1000)), ("softmax 32x1000", softmax(32, 1000))]:
        print("%-34s %8.2f us" % (name, timeit(fn)))
