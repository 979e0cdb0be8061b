"""CPU suite: the conv planner without a device. b200_conv_plan_choose must pick, for every descriptor and switch setting
recorded on the H100 (tests/golden/conv_plans.json.gz, written by tools/make_conv_plan_golden.py), exactly the plan
b200_conv_plan_create built there -- kernel, tile width, grid, k steps, shared memory and split factor -- or the same
refusal; and the int8 ResNet-50 rules refitted on the H100 give the kernels, widths and splits they were measured with."""
import collections
import ctypes as C
import gzip
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "conv_plans.json.gz")
SWITCHES = ("B200_SABER_SPLITK", "B200_SABER_FORCE_BN", "B200_SABER_FORCE_SPLIT", "B200_SABER_SLAB",
            "B200_SABER_PERSISTENT")
H100_SXM_SMS = 132

# int8 ResNet-50 layers at batch 8 with the planner's own choices (no switch set):
# (n, h, w, c, k, r, stride, pad), residual, expected (kernel, block_n, split); None = not pinned
CASES = [
    ((8, 56, 56, 64, 256, 1, 1, 0), True, ("tile", 64, 1)),       # res2 branch2c: was 256 wide
    ((8, 56, 56, 256, 512, 1, 2, 0), False, (None, 64, 1)),       # res3a branch1: was 128 wide
    ((8, 28, 28, 128, 512, 1, 1, 0), True, (None, 64, 1)),        # res3 branch2c: 392 tiles (per-tile or walker)
    ((8, 14, 14, 1024, 256, 1, 1, 0), False, ("tile", 32, 1)),    # res4 branch2a: 64 wide leaves 52 CTAs
    ((8, 14, 14, 1024, 2048, 1, 2, 0), False, ("tile", 64, 1)),   # res5a branch1: 128 CTAs at 64 wide
    ((8, 14, 14, 256, 256, 3, 1, 1), False, ("slab", 64, 1)),     # res4 branch2b: was a 32-wide slab
    ((8, 7, 7, 512, 512, 3, 1, 1), False, ("tile", 64, 2)),       # res5 branch2b: was a 32-wide slab; 392 = 3 x 128 + 8
    ((8, 7, 7, 512, 512, 3, 1, 1), True, ("tile", 64, 2)),        # the same with a residual
    ((1, 7, 7, 512, 512, 3, 1, 1), False, (None, 32, None)),      # b1: the 32-wide plans stay
]


def int8_desc(case, with_res):
    """The descriptor test_conv_plan_gpu.py runs for a CASES entry: u8 in and out, s8 residual, relu."""
    from anakin_b200 import saber_abi as A
    n, h, w, c, k, r, stride, pad = case
    return A.ConvDesc(math=A.MATH_I8, in_dtype=A.UINT8, out_dtype=A.UINT8, res_dtype=A.INT8 if with_res else -1, n=n,
                      h=h, w=w, c=c, k=k, ldc=k, r=r, s=r, pad_h=pad, pad_w=pad, stride_h=stride, stride_w=stride,
                      dil_h=1, dil_w=1, relu=1, sum_scale=0.5)


def golden_records():
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


def set_switches(monkeypatch, env):
    for key in SWITCHES:
        monkeypatch.delenv(key, raising=False)
    for key, value in env.items():
        monkeypatch.setenv(key, value)


def choose(desc, sms):
    """(status, the record fields of the plan b200_conv_plan_choose picks)."""
    from anakin_b200 import saber_abi as A
    out = A.ConvPlanChoice()
    st = A.load().b200_conv_plan_choose(C.byref(desc), sms, C.byref(out))
    if st != A.SUCCESS:
        return st, {}
    return st, {"block_n": out.block_n, "grid_x": out.grid_x, "grid_y": out.grid_y, "k_steps": out.k_steps,
                "smem": out.smem_bytes, "split": out.split, "slab": out.kernel == A.CONV_KERNEL_SLAB,
                "persistent": out.kernel == A.CONV_KERNEL_PERSISTENT}


def test_choose_reproduces_every_recorded_plan(monkeypatch):
    from anakin_b200 import saber_abi as A
    records = golden_records()
    wrong = []
    for rec in records:
        set_switches(monkeypatch, rec["env"])
        st, got = choose(A.ConvDesc(**rec["desc"]), rec["sms"])
        want = {k: rec[k] for k in got}
        if st != rec["status"] or got != want:
            wrong.append((rec["case"], rec["env"], rec["status"], want, st, got))
    assert not wrong, "%d of %d plans differ, first: %s" % (len(wrong), len(records), wrong[:3])


def test_recorded_plans_cover_every_rule_and_switch():
    from anakin_b200 import saber_abi as A
    records = golden_records()
    assert records and all(r["device"].startswith("NVIDIA H100") for r in records)
    reached = collections.defaultdict(set)
    for r in records:
        math = r["desc"]["math"]
        if r["status"] != A.SUCCESS:
            reached[math].add("refusal")
            continue
        kernel = "slab" if r["slab"] else ("persistent" if r["persistent"] else "tile")
        reached[math].add(kernel)
        if r["slab"] and r["desc"]["fuse_pool"]:
            reached[math].add("slab+pool")
        if kernel == "tile" and r["split"] > 1:
            reached[math].add("split%d" % r["split"])
    for math in (A.MATH_I8, A.MATH_F16, A.MATH_TF32X3):
        need = {"tile", "split2", "slab", "slab+pool", "refusal"}
        if math != A.MATH_I8:
            need.add("split4")
        if math != A.MATH_TF32X3:   # (no 3xTF32 walker)
            need.add("persistent")
        assert need <= reached[math], (math, need - reached[math])
    switched = {k for r in records for k in r["env"]}
    assert switched == set(SWITCHES)


def test_retired_math_kind_is_refused(monkeypatch):
    """The retired single-pass tf32 kind (ABI version 1) is refused as unimplemented by the planner, the stem and
    fc_stream, before any of them looks for a device."""
    from anakin_b200 import saber_abi as A
    set_switches(monkeypatch, {})
    lib = A.load()
    fp32 = A.ConvDesc(math=A.MATH_TF32X3, in_dtype=A.FLOAT, out_dtype=A.FLOAT, res_dtype=-1, n=8, h=14, w=14, c=256,
                      k=256, ldc=256, r=3, s=3, pad_h=1, pad_w=1, stride_h=1, stride_w=1, dil_h=1, dil_w=1, relu=1)
    assert choose(fp32, H100_SXM_SMS)[0] == A.SUCCESS
    fp32.math = A.MATH_TF32
    assert choose(fp32, H100_SXM_SMS)[0] == A.UNIMPL_ERROR
    stem = A.StemDesc(math=A.MATH_TF32, out_dtype=A.FLOAT, n=1, c=3, h=224, w=224, k=64, ldc=64, r=7, s=7, stride_h=2,
                      stride_w=2, pad_h=3, pad_w=3, in_inv_scale=1.0)
    out = C.c_int32()
    assert lib.b200_stem_conv_info(C.byref(stem), *[C.byref(out)] * 5) == A.UNIMPL_ERROR
    fc = A.FcStreamDesc(math=A.MATH_TF32, in_dtype=A.FLOAT, out_dtype=A.FLOAT, m=8, k=2048, ldx=2048, n_out=1000, ldo=1000)
    buf = C.create_string_buffer(16)   # never read: the descriptor is refused first
    assert lib.b200_fc_stream_run(C.byref(fc), buf, buf, None, None, buf, None) == A.UNIMPL_ERROR


@pytest.mark.parametrize("case,with_res,expect", CASES)
def test_int8_resnet50_plans_on_h100(case, with_res, expect, monkeypatch):
    set_switches(monkeypatch, {})
    st, got = choose(int8_desc(case, with_res), H100_SXM_SMS)
    assert st == -1
    kernel, bn, split = expect
    got_kernel = "slab" if got["slab"] else ("pers" if got["persistent"] else "tile")
    assert (kernel is None or got_kernel == kernel) and got["block_n"] == bn, got
    assert split is None or got["split"] == split, got
