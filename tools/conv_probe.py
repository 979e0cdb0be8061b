"""Bring-up probe for the wgmma conv kernel: runs a ladder of cases, each in its own
subprocess under a timeout (a deadlocked mbarrier pipeline must not hang the GPU box),
and prints mismatch patterns instead of a bare pass/fail.

  python tools/conv_probe.py            # all cases
  python tools/conv_probe.py --case 3   # one case, in-process
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# name, math, (n,h,w,c,k,r,stride,pad,dil), c_real
CASES = [
    ("i8 1x1 c128 k32 M=128", "i8", (1, 8, 16, 128, 32, 1, 1, 0, 1), 128),
    ("i8 1x1 c64 k64 (SW64)", "i8", (2, 12, 12, 64, 64, 1, 1, 0, 1), 64),
    ("i8 1x1 c32 k64 (SW32)", "i8", (2, 12, 12, 32, 64, 1, 1, 0, 1), 32),
    ("i8 1x1 c16 k64 (no swizzle)", "i8", (2, 12, 12, 16, 64, 1, 1, 0, 1), 16),
    ("i8 3x3 p1 c128 k128", "i8", (2, 14, 14, 128, 128, 3, 1, 1, 1), 128),
    ("i8 3x3 s2 p1 c64 k40", "i8", (1, 24, 24, 64, 40, 3, 2, 1, 1), 64),
    ("i8 7x7 s2 p3 stem c16(3)", "i8", (1, 32, 32, 16, 64, 7, 2, 3, 1), 3),
    ("i8 1x1 c512 k2048 7x7", "i8", (1, 7, 7, 512, 2048, 1, 1, 0, 1), 512),
    ("i8 fc m8 k2048 n1000", "i8", (8, 1, 1, 2048, 1000, 1, 1, 0, 1), 2048),
    ("f16 3x3 p1 c64 k64", "f16", (2, 14, 14, 64, 64, 3, 1, 1, 1), 64),
    ("tf32 3x3 p1 c32 k64", "tf32", (2, 14, 14, 32, 64, 3, 1, 1, 1), 32),
    ("tf32 7x7 stem c4(3)", "tf32", (1, 32, 32, 4, 64, 7, 2, 3, 1), 3),
]


def run_case(idx):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev, pad_channels
    from oracle import pyoracle as O
    name, math, (n, h, w, c, k, r, stride, pad, dil), c_real = CASES[idx]
    rng = np.random.default_rng(idx + 1)
    kw = dict(stride=(stride, stride), pad=(pad, pad), dil=(dil, dil))
    if math == "i8":
        x = rng.integers(-128, 128, (n, h, w, c_real)).astype(np.int8)
        wq = rng.integers(-127, 128, (k, c_real, r, r)).astype(np.int8)
        want = O.conv_s8_nhwc_x86(x, wq, None, None, out_dtype=O.DT_FLOAT, relu=False, **kw)
        run = ConvRunner(A.MATH_I8, (n, h, w, c), A.INT8, wq, None, None, A.FLOAT, relu=False, **kw)
        xin = pad_channels(x, c)
    else:
        x = rng.uniform(-1, 1, (n, h, w, c_real)).astype(np.float32)
        wt = rng.uniform(-1, 1, (k, c_real, r, r)).astype(np.float32)
        if math == "f16":
            xs, ws = x.astype(np.float16), wt.astype(np.float16)
            want = O.conv_f32_nhwc(xs.astype(np.float32), ws.astype(np.float32), None, **kw)
            run = ConvRunner(A.MATH_F16, (n, h, w, c), A.HALF, ws, None, None, A.FLOAT, **kw)
            xin = pad_channels(xs, c)
        else:
            tr = lambda a: (a.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
            want = O.conv_f32_nhwc(tr(x), tr(wt), None, **kw)
            run = ConvRunner(A.MATH_TF32, (n, h, w, c), A.FLOAT, wt, None, None, A.FLOAT, **kw)
            xin = pad_channels(x, c)
    print("case %d: %s  plan=%s" % (idx, name, run.info()), flush=True)
    got = run.run(dev(xin))
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    M = want.shape[0] * want.shape[1] * want.shape[2]
    g2, w2 = got.reshape(M, -1), want.reshape(M, -1)
    diff = np.abs(g2.astype(np.float64) - w2.astype(np.float64))
    tol = 0 if math == "i8" else 1e-3 * max(1.0, np.abs(w2).max())
    bad = diff > tol
    print("  max|diff|=%.6g  max|want|=%.6g  bad=%d/%d" % (diff.max(), np.abs(w2).max(), bad.sum(), bad.size))
    if bad.any():
        rows = np.where(bad.any(axis=1))[0]
        cols = np.where(bad.any(axis=0))[0]
        print("  bad rows: n=%d first=%s" % (len(rows), rows[:24]))
        print("  bad cols: n=%d first=%s" % (len(cols), cols[:24]))
        r0 = rows[0]
        print("  row %d got : %s" % (r0, g2[r0, :8]))
        print("  row %d want: %s" % (r0, w2[r0, :8]))
        print("  row 0 got : %s" % (g2[0, :8],))
        print("  row 0 want: %s" % (w2[0, :8],))
        # does got match some other row of want? (row permutation diagnostics)
        for rr in rows[:3]:
            m = np.where((np.abs(w2 - g2[rr]) <= tol).all(axis=1))[0]
            print("  got row %d equals want rows %s" % (rr, m[:5]))
        return 1
    print("  OK")
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", type=int, default=-1)
    ap.add_argument("--timeout", type=int, default=90)
    a = ap.parse_args()
    if a.case >= 0:
        sys.exit(run_case(a.case))
    fails = 0
    for i in range(len(CASES)):
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--case", str(i)],
                               timeout=a.timeout, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            print(r.stdout, end="")
            if r.returncode != 0:
                fails += 1
                if r.returncode not in (0, 1):
                    print("  exit code %d" % r.returncode)
        except subprocess.TimeoutExpired as e:
            fails += 1
            print("case %d: %s TIMEOUT (%ds)\n%s" % (i, CASES[i][0], a.timeout, (e.stdout or "")[-2000:]))
    print("probe done: %d/%d failed" % (fails, len(CASES)))


if __name__ == "__main__":
    main()
