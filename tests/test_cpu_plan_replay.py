"""CPU suite: the designed data and the fast references of the plan replay (tests/plan_replay.py, run on the GPU by
tests/test_conv_plan_gpu.py::test_recorded_plans_bit_exact).

- Every replayed record's generator keeps its sums exact, checked analytically from the generator's magnitudes.
- On every replayed shape shrunk to one small image (the real c, k, r, s, stride, pooling and kinds), the data meet the
  generators' own bounds and coverage, and the fast references (the float64 accumulator plus the restated fp32
  epilogue, the VNNI int8 oracle) equal the whole-tensor oracle (conv_f32_nhwc, the plain conv_s8_nhwc_x86) bit for bit.
- The records the replay compares reach every kernel, tile width, split, fused pooling, residual path and ragged inner
  product of every math kind, so that a smaller record set or replay fails here instead of going quiet.
"""
import numpy as np
import pytest

import float_exact as F
import plan_replay as R
from anakin_b200 import saber_abi as A
from test_cpu_conv_plan import CASES, int8_desc

GROUPS = R.replay_groups()


def test_replay_groups_hold_every_successful_record():
    recs = R.records()
    ok = [r for r in recs if r["status"] == A.SUCCESS]
    assert sum(len(g) for g in GROUPS.values()) == len(ok) and len(GROUPS) >= 90
    ids = [R.group_id(g) for g in GROUPS.values()]
    assert len(set(ids)) == len(ids), "group ids must be unique"
    # the int8 plans the planner picks on its own at ResNet-50 batch 8 (test_cpu_conv_plan.CASES) are replayed
    descs = [r["desc"] for g in GROUPS.values() for r in g if r["case"].startswith("auto plan")]
    for case, with_res, _ in CASES:
        d = int8_desc(case, with_res)
        assert {f: getattr(d, f) for f, _ in A.ConvDesc._fields_} in descs, case


def test_every_replayed_generator_is_exact():
    """max|X| max|W| times the taps, plus max|residual|, within 2^22 quanta (int8: within the int32 accumulator)."""
    for recs in GROUPS.values():
        for rec in recs:
            R.assert_bound(R.FAMILY[R.kind_of(rec)], rec["desc"])


@pytest.mark.parametrize("family", ["dense", "x3"])
def test_the_bound_check_refuses_larger_magnitudes(family, monkeypatch):
    """At the largest reduction (res5 3x3, c r s = 4608), dense operands one step past the bound, or split-term taps
    per channel one past it, are refused."""
    d = next(r for recs in GROUPS.values() for r in recs if r["case"] == "resnet50 res5_branch2b f16 n8")["desc"]
    kk = R.reduction(d)
    assert kk == 4608
    R.assert_bound(family, d)
    if family == "dense":
        monkeypatch.setattr(F, "dense_magnitude", lambda kk: int(np.sqrt(2 ** F.EXACT_BITS / kk)) + 1)
    else:
        # a tap's three products reach 15 * 15 * 2^10 + 2 * 7 * 15 quanta
        monkeypatch.setattr(R, "x3_taps", lambda desc: 2 ** F.EXACT_BITS // (15 * 15 * 2 ** 10) + 1)
    with pytest.raises(AssertionError, match="not exact"):
        R.assert_bound(family, d)


def shrunk(rec):
    """The record on one small image: n = 1 (fc rows stay, ragged against the row tile), h and w at most 8."""
    d = dict(rec["desc"])
    if d["h"] > 1:
        d["n"] = 1
        d["h"] = d["w"] = min(d["h"], 8)
    return dict(rec, desc=d)


def assert_data_within_bound(family, x, w, res, desc):
    """The data the generator drew stay within the magnitudes bound_units assumes."""
    kk = R.reduction(desc)
    if family == "int8":
        return
    if family == "dense":
        m = F.dense_magnitude(kk)
        assert np.abs(x).max() <= m * 2.0 ** F.DENSE_EX and np.abs(w).max() <= m * 2.0 ** F.DENSE_EW
        assert res is None or np.abs(res).max() <= F.RES_MAX * 2.0 ** (F.DENSE_EX + F.DENSE_EW)
        return
    assert ((w != 0).reshape(w.shape[0], -1).sum(1) <= R.x3_taps(desc)).all()
    for a, e in ((x, F.X3_EX), (w, F.X3_EW)):
        assert np.abs(F.tf32_hi(a)).max() <= 15 * 2.0 ** e and np.abs(F.tf32_lo(a)).max() <= 7 * 2.0 ** (e - 10)
    assert res is None or np.abs(res).max() <= R.X3_RES_MAX * 2.0 ** (F.X3_EX + F.X3_EW - 10)


@pytest.mark.parametrize("shape", list(GROUPS), ids=[R.group_id(recs) for recs in GROUPS.values()])
def test_fast_references_match_the_oracle(shape):
    seen = set()
    for rec, (x, w, bias, scale, res), want in R.replay([shrunk(r) for r in GROUPS[shape]]):
        d, kind = rec["desc"], R.kind_of(rec)
        key = (kind, tuple(sorted(d.items())))
        if key in seen:        # the switch probes share their descriptor
            continue
        seen.add(key)
        family = R.FAMILY[kind]
        x32 = x if family == "int8" else x.astype(np.float32)
        r32 = res if res is None or family == "int8" else res.astype(np.float32)
        assert_data_within_bound(family, x32, w.astype(np.float32) if family != "int8" else w, r32, d)
        if family != "int8":
            if family == "x3":
                ops = F.x3_expected_operands(x32, w)
                quantum = 2.0 ** (F.X3_EX + F.X3_EW - 10)
            else:
                ops, quantum = (x32, w.astype(np.float32)), None
            F.check_conv_exact(*ops, r32, what=R.label(rec), quantum=quantum, **R.conv_kw(d))
        have = R.oracle_expected(kind, x32, w.astype(np.float32) if family != "int8" else w, bias, scale, r32, d)
        assert have.dtype == want.dtype and have.shape == want.shape
        assert np.array_equal(np.ascontiguousarray(have).view(np.uint8), np.ascontiguousarray(want).view(np.uint8)), \
            "%s: the fast reference differs from the oracle" % R.label(rec)


def test_x3_data_separate_every_dropped_term():
    """At a shrunk res5 3x3 shape (k * X3_TAPS < c r s: 9 taps per channel), a missing Alo Whi or Ahi Wlo term, a single
    pass and the full product each change most outputs (float_exact.x3_expected's checks)."""
    rec = shrunk(next(r for recs in GROUPS.values() for r in recs if r["case"] == "resnet50 res5_branch2b tf32x3 n8"))
    d = rec["desc"]
    assert R.x3_taps(d) == 9
    x, w, bias, _ = R.family_data("x3", d)
    F.x3_expected(x, w, bias, d["stride_h"], d["pad_h"], taps=R.x3_taps(d))


def test_replay_reaches_every_kernel_width_split_and_epilogue():
    got = R.reached([r for recs in GROUPS.values() for r in recs])
    for kind in ("int8", "f16", "tf32x3"):
        widths = (32, 64, 128, 256) if kind in ("int8", "f16") else (32, 64, 128)   # fp32 outputs: 128 at most
        need = {"tile%d" % bn for bn in widths} | {"split2", "slab-pool", "slab+pool", "tile+res", "ragged-fc"}
        if kind != "int8":
            need.add("split4")
        if kind != "tf32x3":          # (no 3xTF32 walker)
            need |= {"persistent", "persistent+res"}
        assert need <= got[kind], (kind, sorted(need - got[kind]))
