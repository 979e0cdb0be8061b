"""SE nets on the CPU: graph round trips and fusions, the INT8 Axpy rule, the explicit sigmoid, the gate restatement and
the committed goldens (tests/se_oracle.py is the restatement of anakin_b200/csrc/se.cu)."""
import json
import os
import sys
import tempfile

import numpy as np
import pytest

import se_oracle as S

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _optimised_ops(model, precision):
    """{node: op} of the optimised graph, and whether Graph::save -> load -> Optimize gives the same list. model: a zoo
    name, or a graph dict."""
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build(model, batch=1, precision=precision) if isinstance(model, str) else model
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.Optimize()
    d = [list(x) for x in G.describe()]
    with tempfile.TemporaryDirectory() as t:
        p = os.path.join(t, "g.anakin.bin")
        G.save(p)
        G2 = api.Graph.from_file(p)
    G2.Optimize()
    return {x[0]: x[1] for x in d}, [list(x) for x in G2.describe()] == d


def tiny_se_resnet_with_identity(at, batch=1, precision="fp32"):
    """tiny_se_resnet with an exact identity -- a Scale of weight 1 and bias 0 -- in every block, so that one fusion
    pattern no longer matches: at="gate" puts it between the SE pooling and the squeeze conv (no SqueezeExcite),
    at="axpy" between the Axpy and its ReLU (no AxpyRelu)."""
    from anakin_b200 import modelzoo
    g = modelzoo.build("tiny_se_resnet", batch=batch)
    nodes = {n["name"]: n for n in g["nodes"]}
    for tag in ("res2a", "res2b", "res3a", "res3b"):
        src = tag + "_se_pool" if at == "gate" else tag
        (dst,) = nodes[src]["outs"]
        c = nodes[tag + "_branch2c"]["attrs"]["filter_num"]
        name = src + "_identity"
        g["nodes"].insert(g["nodes"].index(nodes[src]) + 1, {
            "name": name, "op": "Scale", "ins": [src], "outs": [dst],
            "attrs": dict(axis=1, num_axes=1, bias_term=True, weight_1=np.ones((1, c, 1, 1), np.float32),
                          weight_2=np.zeros((1, c, 1, 1), np.float32)),
            "bit_type": None, "lane": 0, "need_wait": False})
        nodes[src]["outs"] = [name]
        nodes[dst]["ins"] = [name if b == src else b for b in nodes[dst]["ins"]]
        g["edges_out"][src] = [(name, None)]
        g["edges_in"][dst] = [(name if b == src else b, s) for b, s in g["edges_in"][dst]]
        g["edges_in"][name] = [(src, None)]
        g["edges_out"][name] = [(dst, None)]
    if precision == "int8":
        modelzoo.apply_int8(g, modelzoo.load_calibration("tiny_se_resnet"))
    return g


@pytest.mark.parametrize("model,blocks", [("tiny_se_resnet", 4), ("se_resnet50", 16)])
def test_parser_round_trip_unfused(model, blocks):
    from anakin_b200 import anakin_bin, modelzoo
    g = modelzoo.build(model, batch=1, centered=False)
    blob = anakin_bin.dumps(g)
    g2 = anakin_bin.loads(blob) if hasattr(anakin_bin, "loads") else None
    ops = [n["op"] for n in g["nodes"]]
    assert ops.count("Axpy") == blocks and ops.count("Activation") == blocks
    if g2 is not None:
        assert [n["name"] for n in g2["nodes"]] == [n["name"] for n in g["nodes"]]
        assert anakin_bin.dumps(g2) == blob


@pytest.mark.parametrize("precision", ["fp32", "int8"])
def test_optimize_fuses_gate_and_axpy_relu(precision):
    ops, same = _optimised_ops("tiny_se_resnet", precision)
    assert same
    assert list(ops.values()).count("SqueezeExcite") == 4 and list(ops.values()).count("AxpyRelu") == 4
    assert ops["res2a_se_pool"] == "SqueezeExcite" and ops["res3b"] == "AxpyRelu"
    assert not {"Axpy", "Activation", "ReLU"} & set(ops.values())


def test_identity_in_the_chain_stops_each_fusion():
    ops, same = _optimised_ops(tiny_se_resnet_with_identity("gate"), "fp32")
    assert same and "SqueezeExcite" not in ops.values() and list(ops.values()).count("Scale") == 4
    assert list(ops.values()).count("Activation") == 4 and list(ops.values()).count("AxpyRelu") == 4
    ops, same = _optimised_ops(tiny_se_resnet_with_identity("axpy"), "fp32")
    assert same and list(ops.values()).count("Axpy") == 4 and list(ops.values()).count("SqueezeExcite") == 4
    assert "AxpyRelu" not in ops.values() and list(ops.values()).count("Scale") == 4


def test_se_resnet50_optimised():
    ops, same = _optimised_ops("se_resnet50", "int8")
    assert same
    assert list(ops.values()).count("SqueezeExcite") == 16 and list(ops.values()).count("AxpyRelu") == 16
    assert "ConvEltwise" not in ops.values()


def axpy_q8_cases():
    """Designed INT8 Axpy data: with ax = ay = 1 and gates 0 / 0.5 / 1 every product is exact, so t lands on chosen
    values -- ties at +-0.5, +-1.5, +-2.5 and both saturation bounds."""
    qx = np.array([1, 3, 5, -1, -3, -5, 127, -128, 100, -100, 0, 2], np.int8)
    qy = np.array([0, 0, 0, 0, 0, 0, 127, -128, 100, -100, 127, -128], np.int8)
    g = np.array([0.5] * 6 + [1.0] * 4 + [0.0, 0.5], np.float32)
    return g, qx, qy


def test_axpy_q8_rule_ties_and_saturation():
    g, qx, qy = axpy_q8_cases()
    t = g * qx.astype(np.float32) + qy.astype(np.float32)
    # coverage of the designed data: ties of both parities and signs, and both bounds exceeded
    assert {0.5, 1.5, 2.5, -0.5, -1.5, -2.5} <= set(t.tolist())
    assert t.max() > 127 and t.min() < -128
    s8 = S.axpy_q8(g[None], qx[None, None, None], qy[None, None, None], 1.0, 1.0, S.DT_INT8)[0, 0, 0]
    assert s8.tolist() == [0, 2, 2, 0, -2, -2, 127, -128, 127, -128, 127, -127]
    # u8 after the ReLU, ay = 2 (exact): the upper bound 255 is exceeded too
    t2 = g * qx.astype(np.float32) + 2 * qy.astype(np.float32)
    assert (t2 > 255).any() and (t2 < 0).any()
    u8 = S.axpy_q8(g[None], qx[None, None, None], qy[None, None, None], 1.0, 2.0, S.DT_UINT8, relu=True)[0, 0, 0]
    assert u8.tolist() == [0, 2, 2, 0, 0, 0, 255, 0, 255, 0, 254, 0]


def test_axpy_factors_carry_u8_factor():
    u = np.float32(127) / np.float32(255)
    ax, ay = S.axpy_factors(0.02, S.DT_INT8, 0.03, S.DT_UINT8, 0.05, S.DT_UINT8)
    assert ax == np.float32(np.float32(0.02) / (np.float32(0.05) * u))
    assert ay == np.float32((np.float32(0.03) * u) / (np.float32(0.05) * u))


def test_axpy_pinned_to_reference_axpy_nv_basic():
    """tests/golden/ref_axpy.json holds what the reference's own naive oracle axpy_nv_basic computed (tools/
    make_ref_axpy_golden.py compiles it from the reference's test file): the restatement matches its input order (gate,
    x, y) and gate index n*C + c bit for bit in the uncontracted form, and the fmaf form the kernel uses lies within
    one rounding of it, on n > 1 and C > 1."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_ref_axpy_golden import case_inputs
    with open(os.path.join(GOLD, "ref_axpy.json")) as f:
        rec = json.load(f)
    assert any(c["shape"][0] > 1 and c["shape"][1] > 1 for c in rec["cases"])
    differ = 0
    for case in rec["cases"]:
        n, c, h, w = case["shape"]
        g, x, y = case_inputs(n, c, h, w, case["seed"])
        ref = np.asarray(case["out_bits"], np.uint32).view(np.float32).reshape(n, c, h, w).transpose(0, 2, 3, 1)
        xn, yn = x.transpose(0, 2, 3, 1), y.transpose(0, 2, 3, 1)
        plain = S.axpy_f32(g, xn, yn, contract=False)
        assert np.array_equal(plain.view(np.uint32), np.ascontiguousarray(ref).view(np.uint32)), case["shape"]
        fused = S.axpy_f32(g, xn, yn)
        gx = np.abs(g[:, None, None, :] * xn).astype(np.float32)
        assert (np.abs(fused - ref) <= np.spacing(gx) + np.spacing(np.abs(ref))).all(), case["shape"]
        differ += int((fused != ref).sum())
    assert differ > 0          # the data makes the contraction visible: the two forms are told apart


def test_fmaf_is_rounded_once():
    from fractions import Fraction
    rng = np.random.default_rng(1)
    a, b, c = (rng.standard_normal(3000).astype(np.float32) for _ in range(3))
    # and sums that land on float32 midpoints: 1 + 2^-24 (+-) tiny
    a = np.concatenate([a, np.float32([1.0, 1.0, 1.0])])
    b = np.concatenate([b, np.float32([2.0 ** -24, 2.0 ** -24, 2.0 ** -24])])
    c = np.concatenate([c, np.float32([1.0, 1.0 + 2.0 ** -23, 3.0])])
    r = S.fmaf(a, b, c)
    for i in range(a.size):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        d = abs(Fraction(float(r[i])) - exact)
        for nb in (np.nextafter(r[i], np.float32(np.inf)), np.nextafter(r[i], np.float32(-np.inf))):
            assert abs(Fraction(float(nb)) - exact) >= d, i


def test_sigmoid_sweep_ulp():
    """The explicit fp32 sigmoid against float64 over a dense sweep of [-90, 90], subnormal outputs included: at most
    2.25 ulp (2.19 measured; the z < 0 branch divides e by 1 + e, and e's rounding sits in a binade below the result's)."""
    z = np.linspace(-90, 90, 2_000_001).astype(np.float32)
    s = S.sigmoid_f32(z).astype(np.float64)
    ref = 1.0 / (1.0 + np.exp(-z.astype(np.float64)))
    ulp = np.spacing(ref.astype(np.float32)).astype(np.float64)
    err = np.abs(s - ref) / ulp
    assert err.max() <= 2.25, float(err.max())
    assert (err <= 1.0).mean() > 0.95
    assert S.sigmoid_f32(np.float32([0.0]))[0] == 0.5 and S.sigmoid_f32(np.float32([-200.0]))[0] == 0.0


@pytest.mark.parametrize("dtype", [S.DT_INT8, S.DT_UINT8, S.DT_FLOAT])
def test_gate_restatement_against_float64(dtype):
    rng = np.random.default_rng(5)
    n, h, w, c, r = 3, 7, 7, 256, 16
    if dtype == S.DT_FLOAT:
        x = rng.standard_normal((n, h, w, c)).astype(np.float32)
        xf, scale = x, 1.0
    else:
        lo, hi = (0, 256) if dtype == S.DT_UINT8 else (-128, 128)
        x = rng.integers(lo, hi, (n, h, w, c)).astype(np.uint8 if dtype == S.DT_UINT8 else np.int8)
        scale = 0.031
        xf = x.astype(np.float64) * scale * (127.0 / 255.0 if dtype == S.DT_UINT8 else 1.0)
    w1 = (rng.standard_normal((r, c)) * np.sqrt(2.0 / c)).astype(np.float32)
    w2 = (rng.standard_normal((c, r)) * np.sqrt(2.0 / r)).astype(np.float32)
    b1 = rng.uniform(-0.1, 0.1, r).astype(np.float32)
    b2 = rng.uniform(-0.1, 0.1, c).astype(np.float32)
    got = S.se_gate(x, dtype, scale, w1, b1, w2, b2)
    want = S.se_gate_f64(xf, w1, b1, w2, b2)
    assert got.dtype == np.float32 and got.shape == (n, c)
    assert np.abs(got - want).max() < 1e-5, float(np.abs(got - want).max())
    assert 0.04 < got.std()      # the gates spread: the data exercises the sigmoid away from its ends


def test_tiny_goldens_regenerate():
    """tests/golden/tiny_se_resnet_* are what tools/make_golden.py computes with the walker, bit for bit."""
    from anakin_b200 import modelzoo
    with open(os.path.join(GOLD, "tiny_se_resnet_calib.json")) as f:
        table = json.load(f)["edge_scales"]
    g = modelzoo.build("tiny_se_resnet", batch=1)
    cal = modelzoo.synthetic_input(8, 32, seed=1000)
    fresh = S.calibrate(g, cal)
    assert {k: float(np.float32(v)) for k, v in fresh.items()} == table
    gold = np.load(os.path.join(GOLD, "tiny_se_resnet_golden.npz"))
    x = modelzoo.synthetic_input(8, 32, seed=42)
    fp32, vals = S.run_fp32(g, x, return_values=True)
    np.testing.assert_array_equal(fp32["prob_out"], gold["prob_fp32"])
    np.testing.assert_array_equal(vals["fc"].reshape(8, -1), gold["logits_fp32"])
    q, trace = S.run_int8(modelzoo.build("tiny_se_resnet", batch=1, precision="int8"), x, table,
                          return_intermediate=True)
    np.testing.assert_array_equal(q["prob_out"], gold["prob_int8"])
    np.testing.assert_array_equal(trace["fc"][0].reshape(8, -1), gold["logits_int8"])
    assert len(set(gold["top1_fp32"].tolist())) >= 3


def test_se_resnet50_fixtures_present():
    from anakin_b200 import modelzoo
    table = modelzoo.load_calibration("se_resnet50")
    g = modelzoo.build("se_resnet50", batch=1, precision="int8")
    # a scale for every INT8 edge: every conv group's output and every Axpy's
    for n in g["nodes"]:
        if n["op"] in ("Convolution", "Axpy"):
            assert n["name"] in table, n["name"]
    gold = np.load(os.path.join(GOLD, "se_resnet50_ref.npz"))
    assert gold["logits_int8"].shape == (32, 1000) and gold["logits_fp32"].shape == (32, 1000)
    assert not os.path.exists(os.path.join(GOLD, "se_resnet50_golden.npz"))
