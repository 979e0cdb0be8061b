"""GPU parity of the conv planner: b200_conv_plan_create builds on the device exactly the plans recorded in
tests/golden/conv_plans.json.gz (which tests/test_cpu_conv_plan.py replays through the device-free planner), and every
recorded plan computes its shape bit for bit on designed data (tests/plan_replay.py): int8 against the CPU oracle (x86
Saber semantics), f16 and tf32x3 on data whose sums are exact, against the oracle's fp32 epilogue."""
import os
import sys

import numpy as np
import pytest

import plan_replay as R
from test_cpu_conv_plan import ROOT, golden_records, set_switches

pytestmark = pytest.mark.gpu

GROUPS = R.replay_groups()
SENTINEL = {R.A.UINT8: 0xA5, R.A.INT8: -91, R.A.HALF: -777.0, R.A.FLOAT: -777.0}
PLAN_FIELDS = ("block_n", "grid_x", "grid_y", "k_steps", "smem", "split", "slab", "persistent")


def test_device_plans_match_the_recorded_plans(monkeypatch):
    import torch
    from anakin_b200 import saber_abi as A
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_conv_plan_golden import cases, record_group
    records = golden_records()
    if any(r["sms"] != torch.cuda.get_device_properties(0).multi_processor_count for r in records):
        pytest.skip("the plans were recorded on a GPU with another SM count")
    wrong = []
    for want, case in zip(records, cases()):
        set_switches(monkeypatch, case[2])
        have = record_group(A.LIB_PATH, [case])[0]
        if have != want:
            wrong.append((want, have))
    assert len(cases()) == len(records) and not wrong, \
        "%d of %d plans differ, first: %s" % (len(wrong), len(records), wrong[:1])


def _runner(rec, w, bias, scale):
    """The record's descriptor as a ConvRunner plan over these weights, bias and scale."""
    from gpu_util import ConvRunner
    d = rec["desc"]
    run = ConvRunner(d["math"], (d["n"], d["h"], d["w"], d["c"]), d["in_dtype"], w, bias, scale, d["out_dtype"],
                     res_dtype=d["res_dtype"], stride=(d["stride_h"], d["stride_w"]), pad=(d["pad_h"], d["pad_w"]),
                     dil=(d["dil_h"], d["dil_w"]), relu=bool(d["relu"]), neg_slope=d["neg_slope"],
                     sum_scale=d["sum_scale"], ldc=d["ldc"], fuse_pool=d["fuse_pool"], pool_stride=d["pool_stride"],
                     pool_pad=d["pool_pad"], pool_floor_as_conv=bool(d["pool_floor_as_conv"]))
    have = {f: getattr(run.d, f) for f, _ in R.A.ConvDesc._fields_}
    assert have == d, (rec["case"], have)
    return run


def _first_differences(got, want, count=3):
    gb = np.ascontiguousarray(got).view(np.dtype("u%d" % got.itemsize))
    wb = np.ascontiguousarray(want).view(np.dtype("u%d" % want.itemsize))
    bad = np.argwhere(gb != wb)
    return bad.shape[0], [(tuple(i), got[tuple(i)].item(), want[tuple(i)].item()) for i in bad[:count]]


@pytest.mark.parametrize("shape", list(GROUPS), ids=[R.group_id(recs) for recs in GROUPS.values()])
def test_recorded_plans_bit_exact(shape, monkeypatch):
    """Every successful record of one shape (every math kind, every switch setting) runs its plan on the kind's designed
    data into a sentinel-filled output of the recorded row pitch, and must give the expected bits everywhere. Where the
    device has the recorded SM count, the plan must also be the recorded one, so that the kernels, widths and splits
    the records claim are the ones that ran."""
    import torch
    from gpu_util import _DT2TORCH, dev, pad_channels
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    wrong, on_device, ran = [], {}, 0
    for rec, (x, w, bias, scale, res), want in R.replay(GROUPS[shape]):
        set_switches(monkeypatch, rec["env"])
        d = rec["desc"]
        for name, a in (("x", x), ("res", res)):
            if a is not None and (name, id(a), d["ldc"]) not in on_device:
                # (the entry keeps the array alive, so that its id stays its own); the residual has the output's pitch
                on_device[name, id(a), d["ldc"]] = (a, dev(a if name == "x" else pad_channels(a, d["ldc"])))
        run = _runner(rec, w, bias, scale)
        info = run.info()
        if rec["sms"] == sms and {f: info[f] for f in PLAN_FIELDS} != {f: rec[f] for f in PLAN_FIELDS}:
            wrong.append("%s: plan %s, recorded %s" % (R.label(rec), info, {f: rec[f] for f in PLAN_FIELDS}))
        out = torch.full((d["n"], run.ho, run.wo, d["ldc"]), SENTINEL[d["out_dtype"]], dtype=_DT2TORCH[d["out_dtype"]],
                         device="cuda")
        run.run(on_device["x", id(x), d["ldc"]][1],
                on_device["res", id(res), d["ldc"]][1] if res is not None else None, out)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        ran += 1
        if (got[..., d["k"]:] != SENTINEL[d["out_dtype"]]).any():
            wrong.append("%s: channels past k lost the sentinel (plan %s)" % (R.label(rec), info))
        got = got[..., :d["k"]]
        assert got.shape == want.shape and got.dtype == want.dtype, (R.label(rec), got.shape, want.shape, got.dtype)
        count, first = _first_differences(got, want)
        if count:
            wrong.append("%s: %d of %d differ, first (index, got, want) %s (plan %s)" % (R.label(rec), count, got.size,
                                                                                      first, info))
    assert ran == len(GROUPS[shape]) and not wrong, "%d failures over %d records:\n%s" % (
        len(wrong), len(GROUPS[shape]), "\n".join(wrong))
