"""SE nets on the H100: the Axpy and SE-gate kernels on designed data, and SE-ResNet in-net against tests/se_oracle.py."""
import os

import numpy as np
import pytest

import se_oracle as S

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _axpy(x, y, g, out_dtype, relu=False, neg_slope=0.0, ax=0.0, ay=0.0, gate_dtype=None):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import _NP2DT, dev, ptr, stream_ptr
    n, h, w, c = x.shape
    d = A.AxpyDesc()
    d.x_dtype, d.y_dtype, d.out_dtype = _NP2DT[x.dtype], _NP2DT[y.dtype], out_dtype
    d.gate_dtype = gate_dtype or A.FLOAT
    d.n, d.hw, d.c, d.ld, d.ldg = n, h * w, c, c, g.shape[1]
    d.relu, d.neg_slope, d.ax, d.ay = int(relu), neg_slope, ax, ay
    xd, yd, gd = dev(x), dev(y), dev(g)
    tdt = {A.FLOAT: torch.float32, A.HALF: torch.float16, A.INT8: torch.int8, A.UINT8: torch.uint8}[out_dtype]
    out = torch.empty(x.shape, dtype=tdt, device="cuda")
    A.check(A.load().b200_axpy_run(d, ptr(gd), ptr(xd), ptr(yd), ptr(out), stream_ptr()), "axpy")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def test_axpy_fp32_fmaf_bit_exact():
    from anakin_b200 import saber_abi as A
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2, 5, 3, 64)).astype(np.float32)
    y = rng.standard_normal((2, 5, 3, 64)).astype(np.float32)
    g = rng.uniform(0, 1, (2, 64)).astype(np.float32)
    # designed: y = -g*x rounded, so that only a single rounding of g*x + y leaves the exact residual
    y[0, 0, 0] = -(g[0] * x[0, 0, 0])
    for relu, slope in ((False, 0.0), (True, 0.0), (True, 0.1)):
        got = _axpy(x, y, g, A.FLOAT, relu, slope)
        want = S.axpy_f32(g, x, y, relu, slope)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), relu
    assert (S.axpy_f32(g, x, y)[0, 0, 0] != 0).any()        # the fma residuals are nonzero: no plain mul + add


def test_axpy_fp16_bit_exact():
    from anakin_b200 import saber_abi as A
    rng = np.random.default_rng(2)
    x = rng.standard_normal((3, 4, 4, 48)).astype(np.float16)
    y = rng.standard_normal((3, 4, 4, 48)).astype(np.float16)
    g = rng.uniform(0, 1, (3, 48)).astype(np.float32)
    got = _axpy(x, y, g, A.HALF, relu=True)
    want = S.axpy_f16(g, x, y, relu=True)
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))


def test_axpy_int8_ties_and_saturation():
    from anakin_b200 import saber_abi as A
    g, qx, qy = [np.tile(a, 16)[: 16 * 12] for a in __import__("test_cpu_se").axpy_q8_cases()]
    c = 16 * 12 // 4
    x = qx.reshape(1, 2, 2, c)
    y = qy.reshape(1, 2, 2, c)
    gg = np.ascontiguousarray(g.reshape(1, 2, 2, c)[:, 0, 0, :])     # one gate row for the four pixels
    for out_dt, relu, ay in ((S.DT_INT8, False, 1.0), (S.DT_UINT8, True, 2.0)):
        got = _axpy(x, y, gg, A.INT8 if out_dt == S.DT_INT8 else A.UINT8, relu, ax=1.0, ay=ay)
        want = S.axpy_q8(gg, x, y, 1.0, ay, out_dt, relu)
        assert np.array_equal(got, want), out_dt
    rng = np.random.default_rng(3)
    x = rng.integers(-128, 128, (2, 3, 5, 32)).astype(np.int8)
    y = rng.integers(0, 256, (2, 3, 5, 32)).astype(np.uint8)
    g = rng.uniform(0, 1, (2, 32)).astype(np.float32)
    ax, ay = S.axpy_factors(0.02, S.DT_INT8, 0.03, S.DT_UINT8, 0.05, S.DT_UINT8)
    got = _axpy(x, y, g, A.UINT8, True, ax=float(ax), ay=float(ay))
    assert np.array_equal(got, S.axpy_q8(g, x, y, ax, ay, S.DT_UINT8, True))


@pytest.mark.parametrize("dtype,n,hw,c", [(S.DT_INT8, 8, 56 * 56, 256), (S.DT_UINT8, 3, 7 * 7, 2048),
                                          (S.DT_INT8, 32, 14 * 14, 1024)])
def test_se_gate_int8_bit_exact(dtype, n, hw, c):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    rng = np.random.default_rng(c + n)
    r = c // 16
    lo, hi = (0, 256) if dtype == S.DT_UINT8 else (-128, 128)
    x = rng.integers(lo, hi, (n, hw, 1, c)).astype(np.uint8 if dtype == S.DT_UINT8 else np.int8)
    w1 = (rng.standard_normal((r, c)) * np.sqrt(2.0 / c)).astype(np.float32)
    w2 = (rng.standard_normal((c, r)) * np.sqrt(2.0 / r)).astype(np.float32)
    b1 = rng.uniform(-0.1, 0.1, r).astype(np.float32)
    b2 = rng.uniform(-0.1, 0.1, c).astype(np.float32)
    d = A.SeGateDesc()
    d.dtype, d.n, d.hw, d.c, d.ld, d.r, d.ldg, d.scale = (A.UINT8 if dtype == S.DT_UINT8 else A.INT8), n, hw, c, c, r, c, 0.03
    lib = A.load()
    ws = torch.zeros(lib.b200_se_gate_workspace_bytes(d), dtype=torch.uint8, device="cuda")
    out = torch.zeros((n, c), dtype=torch.float32, device="cuda")
    W = dev(np.concatenate([w1.ravel(), w2.ravel()]))
    B = dev(np.concatenate([b1, b2]))
    xd = dev(x)
    for _ in range(3):     # repeated launches over the same workspace give the same gate
        A.check(lib.b200_se_gate_run(d, ptr(xd), ptr(W), ptr(B), C_off(W, r * c), C_off(B, r), ptr(out), ptr(ws),
                                     stream_ptr()), "se_gate")
    torch.cuda.synchronize()
    want = S.se_gate(x, dtype, np.float32(0.03), w1, b1, w2, b2)
    got = out.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def C_off(t, elems):
    import ctypes as C
    return C.c_void_p(t.data_ptr() + 4 * elems)


def _optimised(g, batch):
    from anakin_b200 import anakin_bin, api
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return G


def _build(name, batch, precision):
    from anakin_b200 import modelzoo
    g = modelzoo.build(name, batch=batch, precision=precision)
    return g, _optimised(g, batch)


def _valid(arr, info):
    c = info["dims"][1]
    return arr[..., :c] if info["layout"] == 9 else arr


@pytest.mark.parametrize("batch", [1, 4])
def test_tiny_se_resnet_int8_bit_exact(batch, oracle):
    from anakin_b200 import api, modelzoo
    g, G = _build("tiny_se_resnet", batch, "int8")
    scales = {k: float(np.float32(v)) for k, v in modelzoo.load_calibration("tiny_se_resnet").items()}
    x = modelzoo.synthetic_input(batch, 32)
    want, trace = S.run_int8(g, x, scales, return_intermediate=True)
    gates = [d[0] for d in G.describe() if d[1] == "SqueezeExcite"]
    assert len(gates) == 4
    net = api.Net(G, "int8", keep_edges=True, exports=gates)
    net.set_input("input_0", x)
    net.prediction()
    net.sync()
    checked = 0
    for name, op in net.exec_order():
        if name not in trace or op == "SqueezeExcite":
            continue
        arr, info = net.read_tensor(name)
        w_arr, w_dt, _ = trace["pool1" if op.endswith("Pool") else name]
        assert info["dtype"] == w_dt, (name, op, info, w_dt)
        got = _valid(arr, info).reshape(w_arr.shape)
        if w_dt == S.DT_FLOAT:      # the fp32 logits and probabilities of the head
            mr, md = oracle.tensor_cmp(w_arr, got)
            assert md < 1e-5 or mr <= 1e-5, (name, op, mr, md)
        else:
            assert np.array_equal(got, w_arr), (name, op, int((got != w_arr).sum()))
        checked += 1
    assert checked >= 14
    for gname in gates:
        got = net.get_export(gname).reshape(batch, -1)
        want_g = trace[gname][0].reshape(batch, -1)
        assert np.array_equal(got.view(np.uint32), want_g.view(np.uint32)), gname
    assert (net.get_output().argmax(1) == want["prob_out"].argmax(1)).all()


def test_tiny_se_resnet_fp32_and_fp16(oracle):
    from anakin_b200 import api, modelzoo
    batch = 3
    x = modelzoo.synthetic_input(batch, 32)
    g, G = _build("tiny_se_resnet", batch, "fp32")
    want, vals = S.run_fp32(g, x, return_values=True)
    net = api.Net(G, "fp32", keep_edges=True)
    net.set_input("input_0", x)
    net.prediction(); net.sync()
    got = net.get_output()
    mr, md = oracle.tensor_cmp(want["prob_out"], got)
    assert md < 1e-3 or mr <= 1e-3, (mr, md)
    arr, info = net.read_tensor("fc")
    mr, md = oracle.tensor_cmp(vals["fc"].reshape(batch, -1), _valid(arr, info).reshape(batch, -1))
    assert md < 1e-3 or mr <= 1e-3, (mr, md)
    # CUDA-graph replay equals the eager run
    net.prediction(); net.prediction(); net.sync()
    assert net.cuda_graph_active()
    np.testing.assert_array_equal(net.get_output(), got)
    # FP16: every edge tensor is rounded to 11 significant bits; the tiny net holds L = 18 fp16 edges in series (stem, four
    # blocks of branch2a / 2b / 2c / Axpy, the pooling). As for the other FP16 nets (tests/test_net_gpu.py), errors taken
    # as independent: |dlogit| <= 4 * sqrt(L) * 2^-11 * max|logit|, and top-1 equal wherever the margin exceeds twice that
    gold = np.load(os.path.join(GOLD, "tiny_se_resnet_golden.npz"))
    _, G16 = _build("tiny_se_resnet", batch, "fp16")
    net16 = api.Net(G16, "fp16", keep_edges=True)
    net16.set_input("input_0", x)
    net16.prediction(); net16.sync()
    arr, info = net16.read_tensor("fc")
    l16 = _valid(arr, info).reshape(batch, -1).astype(np.float32)
    l32 = gold["logits_fp32"][:batch]
    bound = 4.0 * np.sqrt(18.0) * 2.0 ** -11 * float(np.abs(l32 + gold["logit_offset"]).max())
    assert np.abs(l16 - l32).max() <= bound, (float(np.abs(l16 - l32).max()), bound)
    srt = np.sort(l32, axis=1)
    clear = (srt[:, -1] - srt[:, -2]) > 2 * bound
    assert (net16.get_output().argmax(1)[clear] == gold["top1_fp32"][:batch][clear]).all()


def test_gpu_calibrator_scales_every_int8_edge():
    """anakin_b200/calibrate.py on the FP32 SE net (statistics on the GPU): a scale for every convolution and every
    Axpy output -- the INT8 edges -- equal to the CPU walker's max-abs table up to the float order of the fp32 net."""
    from anakin_b200 import calibrate, modelzoo
    g = modelzoo.build("tiny_se_resnet", batch=8)
    cal = modelzoo.synthetic_input(8, 32, seed=1000)
    table = calibrate.Calibrator(g, calibrate.BatchStream([cal]), algo="maxabs").generate_calibrator_table()
    want = modelzoo.load_calibration("tiny_se_resnet")
    # (the gate chain's interior is fp32 inside the fused SqueezeExcite and needs no scale)
    int8_edges = [n["name"] for n in g["nodes"]
                  if n["op"] in ("Convolution", "Axpy", "ReLU", "Scale", "BatchNorm") and "_se_" not in n["name"]]
    for name in int8_edges:
        assert name in table, name
        assert abs(table[name] - want[name]) <= 1e-3 * want[name], (name, table[name], want[name])
    # the calibrated table runs the INT8 net
    from anakin_b200 import anakin_bin, api
    g8 = modelzoo.apply_int8(modelzoo.build("tiny_se_resnet", batch=2), table)
    G = api.Graph.from_bytes(anakin_bin.dumps(g8))
    G.Optimize()
    net = api.Net(G, "int8")
    net.set_input("input_0", modelzoo.synthetic_input(2, 32))
    net.prediction(); net.sync()
    assert np.isfinite(net.get_output()).all()


def test_se_resnet50_b8():
    from anakin_b200 import api, modelzoo
    gold = np.load(os.path.join(GOLD, "se_resnet50_ref.npz"))
    batch = 8
    x = modelzoo.synthetic_input(batch, 224)
    _, G = _build("se_resnet50", batch, "int8")
    net = api.Net(G, "int8", exports=["fc1000"])
    net.set_input("input_0", x)
    net.prediction(); net.prediction(); net.sync()
    logits = net.get_export("fc1000").reshape(batch, -1)
    np.testing.assert_array_equal(logits, gold["logits_int8"][:batch])
    assert (net.get_output().argmax(1) == gold["top1_int8"][:batch]).all()
    _, G = _build("se_resnet50", batch, "fp32")
    net = api.Net(G, "fp32", exports=["fc1000"])
    net.set_input("input_0", x)
    net.prediction(); net.sync()
    # bench.py's FP32 criterion: max |got - want| <= 2.5e-4 of the largest uncentred logit, and top-1 equal on every
    # image whose top-2 margin exceeds 4 * that error
    want = gold["logits_fp32"][:batch]
    got = net.get_export("fc1000").reshape(batch, -1)
    scale = float(np.abs(want + gold["logit_offset"]).max())
    md = float(np.abs(got - want).max())
    assert md <= 2.5e-4 * scale, (md, scale)
    srt = np.sort(want, axis=1)
    clear = (srt[:, -1] - srt[:, -2]) > 4 * md
    assert (net.get_output().argmax(1)[clear] == gold["top1_fp32"][:batch][clear]).all()


def test_unfused_se_and_axpy_relu_fp32_and_int8_refusal():
    """An identity in the gate chain (or between Axpy and ReLU) keeps the ops unfused: FP32 top-1 is the fused net's,
    and an INT8 net refuses an Axpy whose gate is not a fused SqueezeExcite, naming the node."""
    from anakin_b200 import api, modelzoo
    from test_cpu_se import tiny_se_resnet_with_identity

    def run(g):
        net = api.Net(_optimised(g, 4), "fp32")
        net.set_input("input_0", modelzoo.synthetic_input(4, 32))
        net.prediction(); net.sync()
        return net.get_output().argmax(1).tolist(), {op for _, op in net.exec_order()}

    top, ops = run(modelzoo.build("tiny_se_resnet", batch=4))
    assert {"SqueezeExcite", "AxpyRelu"} <= ops, ops
    for at, fused in (("gate", "SqueezeExcite"), ("axpy", "AxpyRelu")):
        t, o = run(tiny_se_resnet_with_identity(at, batch=4))
        assert fused not in o and "Scale" in o, (at, o)
        assert t == top, (at, t, top)
    G = _optimised(tiny_se_resnet_with_identity("gate", batch=4, precision="int8"), 4)
    with pytest.raises(api.AnakinError, match=r"node res2a \(AxpyRelu\): its gate .* is not a fused SqueezeExcite"):
        api.Net(G, "int8")


def test_worker_two_threads_se_resnet50():
    import tempfile
    from anakin_b200 import anakin_bin, api, modelzoo
    gold = np.load(os.path.join(GOLD, "se_resnet50_ref.npz"))
    batch = 8
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "se_resnet50.anakin.bin")
        anakin_bin.save(modelzoo.build("se_resnet50", batch=batch, precision="int8"), p)
        w = api.Worker(p, "int8", threads=2, batch=batch)
        x = modelzoo.synthetic_input(batch, 224)
        outs = [w.sync_prediction(x, 1000 * batch) for _ in range(4)]
    for o in outs:
        prob = np.asarray(o).reshape(batch, -1)
        assert (prob.argmax(1) == gold["top1_int8"][:batch]).all()
