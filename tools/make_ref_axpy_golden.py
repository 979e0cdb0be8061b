"""Record what the reference's naive Axpy oracle axpy_nv_basic (test/saber/test_saber_axpy.cpp:18-52) computes on
seeded data into tests/golden/ref_axpy.json: shapes, seed and the fp32 output bits. tests/test_cpu_se.py regenerates the
inputs from the seed and checks tests/se_oracle.py's Axpy against these records: input order (gate, x, y), the gate
indexed n*C + c, and the arithmetic.

Needs the reference's sources (REF, default /root/reference): the function template is cut out of the test file (lines
18-52, guarded by a check of its first two lines) into a temporary directory and compiled with tools/ref_shim_axpy.cpp
and -ffp-contract=off, so the record is the uncontracted x * scale + y."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("REF", "/root/reference")
FIRST, LAST = 18, 52
CASES = [(2, 3, 4, 5, 11), (3, 16, 7, 7, 12), (1, 8, 1, 1, 13)]    # n, c, h, w, seed


def case_inputs(n, c, h, w, seed):
    """The seeded NCHW inputs of one case: gate [n][c] in (0, 1), x and y [n][c][h][w] standard normal."""
    rng = np.random.default_rng(seed)
    g = rng.uniform(0, 1, (n, c)).astype(np.float32)
    x = rng.standard_normal((n, c, h, w)).astype(np.float32)
    y = rng.standard_normal((n, c, h, w)).astype(np.float32)
    return g, x, y


def build_ref(tmp):
    src = os.path.join(REF, "test", "saber", "test_saber_axpy.cpp")
    with open(src) as f:
        lines = f.read().split("\n")
    if not lines[FIRST - 1].startswith("template") or "void axpy_nv_basic(" not in lines[FIRST]:
        raise SystemExit("%s:%d is not axpy_nv_basic" % (src, FIRST))
    with open(os.path.join(tmp, "ref_axpy.inc"), "w") as f:
        f.write("\n".join(lines[FIRST - 1:LAST]) + "\n")
    so = os.path.join(tmp, "libref_axpy.so")
    subprocess.run(["g++", "-O2", "-std=c++11", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I" + tmp,
                    os.path.join(ROOT, "tools", "ref_shim_axpy.cpp"), "-o", so], check=True)
    lib = C.CDLL(so)
    lib.ref_axpy_nchw.argtypes = [C.c_void_p] * 4 + [C.c_int] * 4
    return lib


def main():
    out = {"source": "test/saber/test_saber_axpy.cpp:%d-%d axpy_nv_basic" % (FIRST, LAST), "cases": []}
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_ref(tmp)
        for n, c, h, w, seed in CASES:
            g, x, y = case_inputs(n, c, h, w, seed)
            o = np.zeros_like(x)
            lib.ref_axpy_nchw(g.ctypes.data, x.ctypes.data, y.ctypes.data, o.ctypes.data, n, c, h, w)
            out["cases"].append({"shape": [n, c, h, w], "seed": seed, "out_bits": o.view(np.uint32).ravel().tolist()})
    path = os.path.join(ROOT, "tests", "golden", "ref_axpy.json")
    with open(path, "w") as f:
        json.dump(out, f)
        f.write("\n")
    print("wrote %s: %d cases" % (path, len(out["cases"])))


if __name__ == "__main__":
    sys.exit(main())
