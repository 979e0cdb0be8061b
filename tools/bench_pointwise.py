"""Achieved HBM bandwidth of every pointwise / streaming kernel of the library at a bandwidth-sized shape (working set well
above the 50 MB L2), through the C ABI: algorithmic bytes (input + output tensors, weights once) / device time (CUDA events
around back-to-back launches), as a fraction of the measured copy peak (MEASURED_PEAKS.json).
  python tools/bench_pointwise.py                 # table
  ncu --set full -k regex:'pool|softmax|eltwise|activation|scale|nchw|dwconv|fc_stream|conv_stem' -c 40 \
      python tools/bench_pointwise.py --once      # one launch each, for the DRAM-side counters
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from anakin_b200 import saber_abi as A  # noqa: E402
from gpu_util import ptr, stream_ptr  # noqa: E402

lib = None


def rnd(shape, dtype):
    g = torch.Generator(device="cuda").manual_seed(0)
    if dtype in (torch.uint8, torch.int8):
        return torch.randint(0, 120, shape, generator=g, device="cuda", dtype=torch.int32).to(dtype)
    return (torch.rand(shape, generator=g, device="cuda", dtype=torch.float32) * 2 - 1).to(dtype)


def pool_case(n, h, w, c, win, stride, ptype, glob, dtype, tdt, es):
    d = A.PoolDesc()
    d.dtype, d.type, d.n, d.h, d.w, d.c = dtype, ptype, n, h, w, c
    d.window_h = d.window_w = win
    d.stride_h = d.stride_w = stride
    d.global_pooling = int(glob)
    oh, ow = C.c_int32(), C.c_int32()
    lib.b200_pool_out_hw(C.byref(d), C.byref(oh), C.byref(ow))
    x = rnd((n, h, w, c), tdt)
    out = torch.zeros((n, oh.value, ow.value, c), dtype=tdt, device="cuda")
    return (lambda: lib.b200_pool_run(C.byref(d), ptr(x), ptr(out), stream_ptr())), (x.numel() + out.numel()) * es, (x, out, d)


def softmax_case(rows, n):
    x = rnd((rows, n), torch.float32)
    out = torch.empty_like(x)
    return (lambda: lib.b200_softmax_run(ptr(x), ptr(out), rows, n, 1, stream_ptr())), 2 * x.numel() * 4, (x, out)


def eltwise_case(count, dtype, tdt, es):
    a, b = rnd((count,), tdt), rnd((count,), tdt)
    out = torch.empty_like(a)
    return (lambda: lib.b200_eltwise_run(dtype, dtype, dtype, A.ELT_SUM, ptr(a), ptr(b), ptr(out), count, 1.0, 1.0, 1,
                                         stream_ptr())), 3 * count * es, (a, b, out)


def activation_case(count):
    a = rnd((count,), torch.float32)
    out = torch.empty_like(a)
    return (lambda: lib.b200_activation_run(A.FLOAT, A.ACT_RELU, ptr(a), ptr(out), count, 0.0, 0.0, stream_ptr())), 2 * count * 4, (a, out)


def scale_case(pixels, c):
    a = rnd((pixels, c), torch.float32)
    w, b = rnd((c,), torch.float32), rnd((c,), torch.float32)
    out = torch.empty_like(a)
    return (lambda: lib.b200_scale_run(A.FLOAT, ptr(a), ptr(out), pixels, c, ptr(w), ptr(b), stream_ptr())), 2 * a.numel() * 4, (a, w, b, out)


def nchw_case(n, c, h, w, c_pad, out_dtype, tdt, es):
    x = rnd((n, c, h, w), torch.float32)
    out = torch.zeros((n, h, w, c_pad), dtype=tdt, device="cuda")
    return (lambda: lib.b200_nchw_to_nhwc(ptr(x), ptr(out), out_dtype, n, c, h, w, c_pad, 50.0, 0, stream_ptr())), \
        x.numel() * 4 + out.numel() * es, (x, out)


def dwconv_case(n, h, w, c, stride, math, dtype, tdt, es):
    d = A.ConvDesc()
    d.math, d.in_dtype, d.out_dtype, d.res_dtype = math, dtype, dtype, -1
    d.n, d.h, d.w, d.c, d.k, d.ldc, d.r, d.s = n, h, w, c, c, c, 3, 3
    d.pad_h = d.pad_w = 1
    d.stride_h = d.stride_w = stride
    d.dil_h = d.dil_w = 1
    d.relu = 1
    ho = (h + 2 - 3) // stride + 1
    x = rnd((n, h, w, c), tdt)
    wt = rnd((3, 3, c), torch.int8 if es == 1 else tdt)
    b = rnd((c,), torch.float32)
    s = (torch.rand(c, device="cuda") * 1e-3 + 1e-3) if es == 1 else None
    out = torch.zeros((n, ho, ho, c), dtype=tdt, device="cuda")
    return (lambda: lib.b200_dwconv_run(C.byref(d), ptr(x), ptr(wt), ptr(b), ptr(s), ptr(out), stream_ptr())), \
        (x.numel() + out.numel()) * es, (x, wt, b, s, out, d)


def fc_case(m, k, n, math, dtype, tdt, es):
    d = A.FcStreamDesc()
    d.math, d.in_dtype, d.out_dtype = math, dtype, A.FLOAT
    d.m, d.k, d.ldx, d.n_out, d.ldo = m, k, k, n, n
    x = rnd((m, k), tdt)
    w = rnd((n, k), torch.int8 if es == 1 else tdt)
    b = rnd((n,), torch.float32)
    s = (torch.rand(n, device="cuda") * 1e-3 + 1e-3) if es == 1 else None
    out = torch.zeros((m, n), dtype=torch.float32, device="cuda")
    return (lambda: lib.b200_fc_stream_run(C.byref(d), ptr(x), ptr(w), ptr(b), ptr(s), ptr(out), stream_ptr())), \
        w.numel() * es + x.numel() * es + out.numel() * 4, (x, w, b, s, out, d)


def stem_case(n):
    d = A.StemDesc()
    d.math, d.out_dtype = A.MATH_I8, A.UINT8
    d.n, d.c, d.h, d.w, d.k, d.ldc = n, 3, 224, 224, 64, 64
    d.r, d.s, d.stride_h, d.stride_w, d.pad_h, d.pad_w = 7, 7, 2, 2, 3, 3
    d.relu, d.in_inv_scale, d.monotone_epilogue = 1, 50.0, 1
    d.fuse_pool, d.pool_type = 1, A.POOL_MAX
    d.pool_window_h = d.pool_window_w = 3
    d.pool_stride_h = d.pool_stride_w = 2
    wq = np.random.default_rng(0).integers(-127, 128, (64, 3, 7, 7)).astype(np.int8)
    packed = np.zeros(lib.b200_stem_packed_weight_bytes(C.byref(d)), np.uint8)
    lib.b200_stem_pack_weights(C.byref(d), wq.ctypes.data_as(C.c_void_p), packed.ctypes.data_as(C.c_void_p))
    x = rnd((n, 3, 224, 224), torch.float32)
    wd = torch.from_numpy(packed).cuda()
    b = rnd((64,), torch.float32)
    s = torch.rand(64, device="cuda") * 1e-3 + 1e-3
    out = torch.zeros((n, 56, 56, 64), dtype=torch.uint8, device="cuda")
    return (lambda: lib.b200_stem_conv_run(C.byref(d), ptr(x), ptr(wd), ptr(b), ptr(s), ptr(out), stream_ptr())), \
        x.numel() * 4 + out.numel(), (x, wd, b, s, out, d)


def timeit(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3


def main():
    global lib
    ap = argparse.ArgumentParser()
    ap.add_argument("--once", action="store_true", help="one launch per kernel (under ncu)")
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    lib = A.load()
    peak = 6581.6
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peak = json.load(open(p))["hbm_gbs"]
    cases = [
        ("pool_q8_simd 3x3/s2 max  u8 256x112x112x64", lambda: pool_case(256, 112, 112, 64, 3, 2, 1, False, A.UINT8, torch.uint8, 1)),
        ("pool_f32     2x2/s2 max  f32 32x224x224x64", lambda: pool_case(32, 224, 224, 64, 2, 2, 1, False, A.FLOAT, torch.float32, 4)),
        ("pool_f16     3x3/s2 max  f16 128x112x112x64", lambda: pool_case(128, 112, 112, 64, 3, 2, 1, False, A.HALF, torch.float16, 2)),
        ("pool global avg          u8 4096x7x7x2048", lambda: pool_case(4096, 7, 7, 2048, 7, 1, 2, True, A.UINT8, torch.uint8, 1)),
        ("softmax_rows             f32 65536x1000", lambda: softmax_case(65536, 1000)),
        ("eltwise_q8 sum+relu      u8 256M", lambda: eltwise_case(256 << 20, A.UINT8, torch.uint8, 1)),
        ("eltwise_f32 sum+relu     f32 64M", lambda: eltwise_case(64 << 20, A.FLOAT, torch.float32, 4)),
        ("activation_f32 relu      f32 96M", lambda: activation_case(96 << 20)),
        ("scale_f32                f32 1.5M x 64", lambda: scale_case(3 << 19, 64)),
        ("nchw_to_nhwc fp32->s8    256x3x224x224 -> c16", lambda: nchw_case(256, 3, 224, 224, 16, A.INT8, torch.int8, 1)),
        ("dwconv f16 3x3/s1        128x112x112x64", lambda: dwconv_case(128, 112, 112, 64, 1, A.MATH_F16, A.HALF, torch.float16, 2)),
        ("dwconv int8 3x3/s1       256x112x112x64", lambda: dwconv_case(256, 112, 112, 64, 1, A.MATH_I8, A.UINT8, torch.uint8, 1)),
        ("fc_stream fp32 (VGG fc6) m4 k25088 n4096", lambda: fc_case(4, 25088, 4096, A.MATH_TF32X3, A.FLOAT, torch.float32, 4)),
        ("fc_stream int8           m8 k25088 n4096", lambda: fc_case(8, 25088, 4096, A.MATH_I8, A.UINT8, torch.uint8, 1)),
        ("conv_stem int8 7x7/s2 + pool 3x3/s2  256 imgs", lambda: stem_case(256)),
    ]
    print("%-52s %10s %10s %9s %7s" % ("kernel / shape", "MB", "us", "GB/s", "of peak"))
    for name, mk in cases:
        fn, nbytes, keep = mk()
        if a.once:
            fn()
            torch.cuda.synchronize()
            print("%-52s %10.1f" % (name, nbytes / 1e6))
        else:
            t = timeit(fn, a.reps)
            gbs = nbytes / t / 1e9
            print("%-52s %10.1f %10.1f %9.0f %6.1f%%" % (name, nbytes / 1e6, t * 1e6, gbs, 100 * gbs / peak))
        del keep, fn
        torch.cuda.empty_cache()
    print("peak = %.1f GB/s (measured device copy, MEASURED_PEAKS.json)" % peak)


if __name__ == "__main__":
    main()
