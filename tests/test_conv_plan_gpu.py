"""GPU parity of the conv planner: b200_conv_plan_create builds on the device exactly the plans recorded in
tests/golden/conv_plans.json.gz (which tests/test_cpu_conv_plan.py replays through the device-free planner), and the int8
plans the planner picks on its own for the ResNet-50 layer shapes at batch 8 are bit-exact against the CPU oracle
(x86 Saber semantics). The kernel, tile width and split each of those shapes gets are pinned in test_cpu_conv_plan.py."""
import os
import sys

import numpy as np
import pytest

from test_cpu_conv_plan import CASES, ROOT, golden_records, set_switches

pytestmark = pytest.mark.gpu


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


# (expect, the plan of each shape, is checked by test_cpu_conv_plan.py; the cases keep their ids here)
@pytest.mark.parametrize("case,with_res,expect", CASES)
def test_conv_int8_auto_plan_bit_exact(case, with_res, expect, oracle, monkeypatch):
    set_switches(monkeypatch, {})
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev, pad_channels
    n, h, w, c, k, r, stride, pad = case
    rng = np.random.default_rng(hash((case, with_res)) % (2 ** 31))
    x = rng.integers(0, 256, (n, h, w, c)).astype(np.uint8)
    wq = rng.integers(-127, 128, (k, c, r, r)).astype(np.int8)
    bias = rng.uniform(-2000, 2000, k).astype(np.float32)
    scale = rng.uniform(1e-4, 4e-4, k).astype(np.float32)
    kw = dict(stride=(stride, stride), pad=(pad, pad), dil=(1, 1), relu=True)
    oh = oracle.conv_out_size(h, pad, 1, r, stride)
    res = rng.integers(-128, 128, (n, oh, oh, k)).astype(np.int8) if with_res else None
    out_dtype = A.UINT8
    want = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, residual=res, sum_scale=0.5, out_dtype=out_dtype, **kw)
    run = ConvRunner(A.MATH_I8, x.shape, A.UINT8, wq, bias, scale, out_dtype,
                     res_dtype=(A.INT8 if with_res else -1), sum_scale=0.5, ldc=k, **kw)
    got = run.run(dev(x), dev(pad_channels(res, k)) if with_res else None)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.cpu().numpy(), want)
