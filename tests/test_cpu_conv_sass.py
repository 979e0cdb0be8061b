"""CPU suite: the 8-bit wgmma convolutions issue their MMAs back to back.

wgmma is asynchronous: a warpgroup can queue the MMAs of a whole filter row (slab kernel) or k stage (im2col kernel)
and let the tensor cores run them while it moves on. ptxas keeps that only for a straight run of wgmma instructions.
Put a branch between two of them -- a runtime loop around one MMA, or a runtime choice of the s8 / u8 instruction at
every MMA -- and each one is issued on its own, behind a WARPGROUP.ARRIVE. These tests read the SASS of the built
library (cuobjdump) and check, for every 8-bit instance of the two kernels, that the MMAs of one row or stage follow
one another with no BRA, WARPGROUP.ARRIVE or WARPGROUP.DEPBAR between them, once per A-operand type."""
import collections
import gzip
import json
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "anakin_b200", "lib", "libb200saber.so")

KIND_I8, KIND_E4M3 = 0, 4
MATH_TF32X3 = 3
ELEM_BYTES = {0: 1, 1: 2, 2: 4, 3: 4, 4: 1}   # operand bytes per element of each math kind


def _cuobjdump():
    found = shutil.which("cuobjdump")
    if found:
        return found
    home = os.environ.get("CUDA_HOME") or os.environ.get("CUDA_PATH") or "/usr/local/cuda"
    path = os.path.join(home, "bin", "cuobjdump")
    return path if os.access(path, os.X_OK) else None


@pytest.fixture(scope="module")
def sass():
    """mangled kernel name -> list of its SASS instructions (opcode and operands, without addresses or encodings)"""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump is not installed")
    assert os.path.exists(LIB), "build the library first: %s" % LIB
    text = subprocess.run([tool, "-sass", LIB], check=True, stdout=subprocess.PIPE, text=True).stdout
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if m and cur is not None:
            cur.append(m.group(1))
    return funcs


def _mma_runs(instrs):
    """{MMA type: lengths of its straight runs, longest first}. A run is a sequence of MMAs of one type with no branch,
    warpgroup arrive or warpgroup wait between them (address arithmetic may sit in between)."""
    runs = collections.defaultdict(list)
    key, n = None, 0
    for ins in instrs:
        op = re.sub(r"^@!?U?P\w+\s+", "", ins).split()[0]
        m = re.match(r"[IQH]GMMA\.", op)
        if m and op == key:
            n += 1
            continue
        if key is not None and (m or op.startswith(("BRA", "WARPGROUP.ARRIVE", "WARPGROUP.DEPBAR"))):
            runs[key].append(n)
            key, n = None, 0
        if m:
            key, n = op, 1
    if key is not None:
        runs[key].append(n)
    return {k: sorted(v, reverse=True) for k, v in runs.items()}


def _instances(sass, kernel):
    """(kind, BN, mangled name) of every 8-bit instance of `kernel`"""
    out = []
    for name in sass:
        m = re.match(r"_ZN4b200\d+%sILi(\d+)ELi(\d+)E" % kernel, name)
        if m and int(m.group(1)) in (KIND_I8, KIND_E4M3):
            out.append((int(m.group(1)), int(m.group(2)), name))
    return sorted(out)


def _mma_types(kind, bn):
    ni = min(bn, 128)
    if kind == KIND_I8:   # unsigned (post-ReLU) and signed activations, both against signed weights
        return ["IGMMA.64x%dx32.U8.S8" % ni, "IGMMA.64x%dx32.S8.S8" % ni]
    return ["QGMMA.64x%dx32.F32.E4M3.E4M3" % ni]


def test_slab_kernel_issues_each_filter_row_back_to_back(sass):
    # a 3-tap filter row is 3 x 2 k slices (64-byte channel chunks) or 3 x 4 (128-byte chunks), per 128-wide N block
    inst = _instances(sass, "conv_slab_kernel")
    assert len(inst) == 8, inst
    for kind, bn, name in inst:
        nb = max(1, bn // 128)
        runs = _mma_runs(sass[name])
        for t in _mma_types(kind, bn):
            got = runs.get(t, [])
            assert len(got) >= 2 and got[0] >= 12 * nb and got[1] >= 6 * nb, \
                "slab kind %d BN %d: %s runs %s" % (kind, bn, t, got[:4])


def test_im2col_kernel_issues_each_stage_back_to_back(sass):
    # a stage is 4 k slices of 32 bytes, per 128-wide N block
    inst = _instances(sass, "conv_igemm_kernel")
    assert len(inst) >= 8, inst
    for kind, bn, name in inst:
        nb = max(1, bn // 128)
        runs = _mma_runs(sass[name])
        for t in _mma_types(kind, bn):
            got = runs.get(t, [])
            assert got and got[0] >= 4 * nb, "im2col kind %d BN %d: %s runs %s" % (kind, bn, t, got[:4])


def test_every_recorded_slab_plan_takes_an_unrolled_row():
    # The slab kernel's unrolled rows cover 3 taps of 64- or 128-byte channel chunks; other geometries (5x5 / 7x7
    # filters, 32-byte chunks) and 3xTF32 take its runtime loop. No recorded plan of a zoo net may land there unnoticed.
    with gzip.open(os.path.join(ROOT, "tests", "golden", "conv_plans.json.gz"), "rt") as f:
        plans = [e for e in json.load(f) if e.get("slab")]
    assert plans
    for e in plans:
        d = e["desc"]
        if d["math"] == MATH_TF32X3:
            continue
        c_bytes = d["c"] * ELEM_BYTES[d["math"]]
        chunk = next(x for x in (128, 64, 32, 16) if c_bytes % x == 0)   # conv_common.cuh pick_chunk
        assert (d["s"], chunk) in ((3, 64), (3, 128)), "%s: s %d, %d-byte chunks" % (e["case"], d["s"], chunk)
