"""Device time of b200_head_run / b200_fc_stream_run variants (CUDA events over back-to-back launches)."""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from anakin_b200 import saber_abi as A   # noqa: E402
from gpu_util import dev, ptr, stream_ptr   # noqa: E402

lib = A.load()


def timeit(fn, reps=50):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def head(m, hw, c, n, softmax=True):
    side = int(round(hw ** 0.5))
    x = dev(np.random.randint(0, 256, (m, side, side, c)).astype(np.uint8))
    w = dev(np.random.randint(-127, 128, (n, c)).astype(np.int8))
    b, s = dev(np.zeros(n, np.float32)), dev(np.full(n, 1e-4, np.float32))
    ldo = (n + 3) // 4 * 4
    fd = A.FcStreamDesc()
    fd.math, fd.in_dtype, fd.out_dtype = A.MATH_I8, A.UINT8, A.FLOAT
    fd.m, fd.k, fd.ldx, fd.n_out, fd.ldo = m, c, c, n, ldo
    hd = A.HeadDesc()
    hd.fc, hd.hw, hd.pool_max, hd.ldp = fd, hw, 0, ldo
    pooled = torch.zeros((m, c), dtype=torch.uint8, device="cuda")
    logits = torch.zeros((m, ldo), dtype=torch.float32, device="cuda")
    prob = torch.zeros((m, ldo), dtype=torch.float32, device="cuda")
    bar = torch.zeros(lib.b200_head_workspace_bytes(C.byref(hd)), dtype=torch.uint8, device="cuda")
    sp = stream_ptr()
    f = lambda: lib.b200_head_run(C.byref(hd), ptr(x), ptr(pooled), ptr(w), ptr(b), ptr(s), ptr(logits),
                                  ptr(prob) if softmax else None, ptr(bar), sp)
    return timeit(f)


def fc(m, k, n, math):
    if math == "i8":
        x, w = dev(np.random.randint(0, 256, (m, k)).astype(np.uint8)), dev(np.random.randint(-127, 128, (n, k)).astype(np.int8))
        mk, dt, es = A.MATH_I8, A.UINT8, 1
        s = dev(np.full(n, 1e-4, np.float32))
    else:
        x, w = dev(np.random.rand(m, k).astype(np.float32)), dev(np.random.rand(n, k).astype(np.float32))
        mk, dt, es, s = A.MATH_TF32X3, A.FLOAT, 4, None
    b = dev(np.zeros(n, np.float32))
    fd = A.FcStreamDesc()
    fd.math, fd.in_dtype, fd.out_dtype = mk, dt, A.FLOAT
    fd.m, fd.k, fd.ldx, fd.n_out, fd.ldo = m, k, k, n, n
    out = torch.zeros((m, n), dtype=torch.float32, device="cuda")
    sp = stream_ptr()
    f = lambda: lib.b200_fc_stream_run(C.byref(fd), ptr(x), ptr(w), ptr(b), ptr(s), ptr(out), sp)
    us = timeit(f, 20)
    return us, n * k * es / us / 1e3


if __name__ == "__main__":
    print("head 8x49x2048->1000 with softmax  %.1f us" % head(8, 49, 2048, 1000, True))
    print("head 8x49x2048->1000 no softmax    %.1f us" % head(8, 49, 2048, 1000, False))
    print("head 8x1x2048->1000 no softmax     %.1f us" % head(8, 1, 2048, 1000, False))
    print("head 8x1x256->64 no softmax        %.1f us" % head(8, 1, 256, 64, False))
    for m, k, n, math in [(8, 2048, 1000, "i8"), (4, 25088, 4096, "f32"), (4, 4096, 4096, "f32"), (4, 4096, 1000, "f32")]:
        us, gbs = fc(m, k, n, math)
        print("fc_stream %s m%d k%d n%d  %.1f us  %.0f GB/s of weights" % (math, m, k, n, us, gbs))
