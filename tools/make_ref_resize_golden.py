"""Record what the reference's x86 BILINEAR_NO_ALIGN resize computes for every case of
tests/image_resize_oracle.py::REF_CASES into tests/golden/ref_resize.json: the fp32 result of resizing the case's image
to (rh, rw) and cropping (top, left, out_h, out_w), as [shape, dtype, SHA-256]. tests/test_cpu_image_resize.py checks the
numpy oracle's fp32 stage against these records.

Needs the reference's sources (REF, default /root/reference): resize_bilinear_no_align_kernel is cut out of
saber/funcs/impl/x86/saber_resize.cpp (lines 103-153, guarded by a grep of the first line) into a temporary directory
and compiled with tools/ref_shim_resize.cpp and -ffp-contract=off."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("REF", "/root/reference")
FIRST, LAST = 103, 153


def build_ref(tmp):
    src = os.path.join(REF, "saber", "funcs", "impl", "x86", "saber_resize.cpp")
    with open(src) as f:
        lines = f.read().split("\n")
    if "template<typename dtype>" not in lines[FIRST - 1] or "resize_bilinear_no_align_kernel" not in lines[FIRST]:
        raise SystemExit("%s:%d is not resize_bilinear_no_align_kernel" % (src, FIRST))
    with open(os.path.join(tmp, "ref_resize.inc"), "w") as f:
        f.write("\n".join(lines[FIRST - 1:LAST]) + "\n")
    so = os.path.join(tmp, "libref_resize.so")
    subprocess.run(["g++", "-O2", "-std=c++11", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I" + tmp,
                    os.path.join(ROOT, "tools", "ref_shim_resize.cpp"), "-o", so], check=True)
    lib = C.CDLL(so)
    lib.ref_resize_bilinear_no_align_hwc.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    return lib


def digest(a):
    a = np.ascontiguousarray(a)
    return [list(a.shape), str(a.dtype), hashlib.sha256(a.tobytes()).hexdigest()]


def main():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import image_resize_oracle as O
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_ref(tmp)
        for case in O.REF_CASES:
            h, w, c, s, oh, ow, _ = case
            rh, rw, top, left = O.geometry(h, w, s, oh, ow)
            src = O.ref_case_image(case).astype(np.float32)
            full = np.zeros((rh, rw, c), np.float32)
            lib.ref_resize_bilinear_no_align_hwc(src.ctypes.data, h, w, c, full.ctypes.data, rh, rw)
            ref = full[top:top + oh, left:left + ow]
            _, mine = O.image_resize_u8(O.ref_case_image(case), s, oh, ow, return_float=True)
            same = np.array_equal(ref.view(np.uint32), mine.view(np.uint32))
            print("%-32s rh x rw %5d x %5d  oracle %s" % (O.ref_case_key(case), rh, rw, "equal" if same else "DIFFERS"))
            out[O.ref_case_key(case)] = digest(ref)
    path = os.path.join(ROOT, "tests", "golden", "ref_resize.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote %s: %d records" % (path, len(out)))


if __name__ == "__main__":
    main()
