"""End-to-end GPU parity: Net<NV,P>::prediction() (C++ framework over the CUDA C ABI) against
the model-level CPU oracle (oracle/model_walker.py) on the same seeded model and inputs.

  FP32 : reference criterion (test_saber_base.h:470 / tensor_cmp_host) at 1e-3 on the
         softmax output and on the logits.
  INT8 : every int8 edge tensor bit-exact against the x86-semantics oracle, logits equal,
         top-1 identical (BASELINE north_star: "exact top-1 class index for INT8").
"""
import os
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _build(name, batch, precision):
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build(name, batch=batch, precision=precision)
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return g, G


def _run(G, precision, x, graph=True, keep_edges=True):
    """keep_edges: one buffer per edge, so that intermediate tensors can be read back after prediction()."""
    from anakin_b200 import api
    net = api.Net(G, precision, keep_edges=keep_edges)
    if not graph:
        net.set_cuda_graph(False)
    net.set_input("input_0", x)
    net.prediction()
    net.sync()
    return net


def _check_fp32_logits(oracle, want, got, what, offset):
    """BASELINE.md section 3 on the LOGITS (the probabilities of a 1000-way softmax are ~1e-3 and would pass anything).
    Compared are the logits with the centring offset added back (`logit_offset` of the golden file: the same constant
    vector on both sides) -- the magnitudes the network actually accumulates, which is what a relative error refers to:
      1. the reference metric tensor_cmp_host (tensor_op.cpp:580-599) at 1e-3, as the reference applies it;
      2. max-norm error <= 2.5e-4 of the largest |logit|;
      3. per element |a-b| <= 1e-3 * max(|a|,|b|) for every logit above 20 % of the largest one (a logit that happens
         to sit near zero moves by more than 1e-3 of itself as soon as the same fp32 products are summed in another
         order, so no second implementation can meet a scale-free bound on ALL elements);
      4. at least 90 % of all elements meet the scale-free |a-b| / max(|a|,|b|,1e-6) <= 1e-3 as well."""
    want = np.asarray(want, np.float32) + offset
    got = np.asarray(got, np.float32) + offset
    assert want.shape == got.shape, (want.shape, got.shape)
    mr, md = oracle.tensor_cmp(want, got)
    assert md < 1e-3 or mr <= 1e-3, (what, mr, md)
    scale = float(np.abs(want).max())
    diff = np.abs(want - got)
    assert diff.max() <= 2.5e-4 * scale, (what, float(diff.max()), scale)
    mag = np.maximum(np.abs(want), np.abs(got))
    big = mag >= 0.2 * scale
    assert big.any() and (diff[big] / mag[big]).max() <= 1e-3, (what, float((diff[big] / mag[big]).max()))
    strict = diff / np.maximum(mag, 1e-6)
    assert (strict <= 1e-3).mean() >= 0.90, (what, float((strict <= 1e-3).mean()))
    return float(diff.max()), scale


def _logits(net, node, batch):
    arr, info = net.read_tensor(node)
    return _valid(arr, info).reshape(batch, -1)


def _valid(arr, info):
    c = info["dims"][1]
    return arr[..., :c] if info["layout"] == 9 else arr


@pytest.mark.parametrize("batch", [1, 3])
def test_tiny_resnet_fp32(batch, oracle):
    from anakin_b200 import modelzoo
    from oracle import model_walker as W
    g, G = _build("tiny_resnet", batch, "fp32")
    x = modelzoo.synthetic_input(batch, 32)
    want = W.run_fp32(g, x)["prob_out"]
    net = _run(G, "fp32", x)
    got = net.get_output()
    mr, md = oracle.tensor_cmp(want, got)
    assert md < 1e-3 or mr <= 1e-3, (mr, md)
    assert (got.argmax(1) == want.argmax(1)).all()
    # second + third call exercise the CUDA-graph replay path and must give the same answer
    net.prediction(); net.prediction(); net.sync()
    assert net.cuda_graph_active()
    np.testing.assert_array_equal(net.get_output(), got)


@pytest.mark.parametrize("batch", [1, 4])
@pytest.mark.parametrize("model", ["tiny_resnet", "tiny_mobilenet"])
def test_tiny_nets_int8_bit_exact(model, batch, oracle):
    """Every int8 edge of the net against the x86-semantics oracle. tiny_mobilenet: the INT8 depthwise kernel
    (SaberDepthWiseConv's INT8 arm) and the stem kernel without a pooling, in-net."""
    from anakin_b200 import modelzoo
    from oracle import model_walker as W
    g, G = _build(model, batch, "int8")
    scales = {k: float(np.float32(v)) for k, v in modelzoo.load_calibration(model).items()}
    x = modelzoo.synthetic_input(batch, 32)
    want, trace = W.run_int8(g, x, scales, return_intermediate=True)
    net = _run(G, "int8", x)
    checked = 0
    for name, op in net.exec_order():
        if name not in trace:
            continue
        arr, info = net.read_tensor(name)
        # a conv that absorbed its MAX pooling (INT8 too: one launch of the stem kernel) holds the pooled tensor
        w_arr, w_dt, w_scale = trace["pool1" if op.endswith("Pool") else name]
        assert info["dtype"] == w_dt, (name, op, info, w_dt)
        got = _valid(arr, info)
        if w_arr.ndim == 4 and got.shape != w_arr.shape:
            got = got.reshape(w_arr.shape)
        if w_dt == 1:
            mr, md = oracle.tensor_cmp(w_arr, got)
            assert md < 1e-5 or mr <= 1e-5, (name, op, mr, md)
        else:
            bad = np.argwhere(got != w_arr)
            assert bad.shape[0] == 0, "%s (%s): %d mismatching codes, first %s" % (name, op, bad.shape[0], bad[:3])
        checked += 1
    assert checked >= 10
    got = net.get_output()
    assert (got.argmax(1) == want["prob_out"].argmax(1)).all()
    mr, md = oracle.tensor_cmp(want["prob_out"], got)
    assert md < 1e-5 or mr <= 1e-5


def test_tiny_resnet_golden_fixture():
    """Committed oracle outputs (tools/make_golden.py) -- does not need /root/reference."""
    from anakin_b200 import modelzoo
    from oracle import pyoracle as O
    gold = np.load(os.path.join(GOLD, "tiny_resnet_golden.npz"))
    nb = gold["top1_int8"].shape[0]
    assert len(set(gold["top1_fp32"].tolist())) >= 3      # the fixture discriminates: several classes win
    g, G = _build("tiny_resnet", nb, "int8")
    net = _run(G, "int8", modelzoo.synthetic_input(nb, 32))
    got = net.get_output()
    assert (got.argmax(1) == gold["top1_int8"]).all()
    np.testing.assert_array_equal(_logits(net, "fc", nb), gold["logits_int8"])
    np.testing.assert_allclose(got, gold["prob_int8"], rtol=1e-4, atol=1e-6)
    g, G = _build("tiny_resnet", nb, "fp32")
    net = _run(G, "fp32", modelzoo.synthetic_input(nb, 32))
    _check_fp32_logits(O, gold["logits_fp32"], _logits(net, "fc", nb), "tiny_resnet fp32", gold["logit_offset"])
    assert (net.get_output().argmax(1) == gold["top1_fp32"]).all()


def test_resnet50_int8_golden_and_oracle(oracle):
    from anakin_b200 import modelzoo
    from oracle import model_walker as W
    batch = 2
    gold = np.load(os.path.join(GOLD, "resnet50_golden.npz"))
    g, G = _build("resnet50", batch, "int8")
    x = modelzoo.synthetic_input(batch)
    net = _run(G, "int8", x)
    got = net.get_output()
    assert (got.argmax(1) == gold["top1_int8"][:batch]).all()
    logits, info = net.read_tensor("fc1000")
    np.testing.assert_array_equal(_valid(logits, info).reshape(batch, -1), gold["logits_int8"][:batch])
    # full-depth bit-exactness of a late int8 edge against a fresh oracle run
    scales = {k: float(np.float32(v)) for k, v in modelzoo.load_calibration("resnet50").items()}
    want, trace = W.run_int8(g, x, scales, return_intermediate=True)
    # (conv1 absorbs pool1 -- one launch of the stem kernel -- so the tensor of node conv1 is the oracle's pool1)
    for node, oracle_node in (("conv1", "pool1"), ("res2a_branch2c",) * 2, ("res3d_branch2c",) * 2, ("res5c_branch2c",) * 2,
                              ("pool5",) * 2):
        arr, info = net.read_tensor(node)
        want_t = trace[oracle_node][0]
        np.testing.assert_array_equal(_valid(arr, info).reshape(want_t.shape), want_t, err_msg=node)
    assert net.launched_ops() <= 60


@pytest.mark.parametrize("batch", [8, 32])
def test_resnet50_int8_full_batch_matches_golden_and_is_batch_invariant(batch):
    """BASELINE.json's full sizes (batch 8 and 32: other tile widths, split-K factors and wave counts than the
    batch-2 plans the oracle pins): images are independent, so image i of the big batch must give bit-for-bit the
    logits it gives in a batch of 4 -- which are the committed golden logits for the first four."""
    from anakin_b200 import modelzoo
    gold = np.load(os.path.join(GOLD, "resnet50_golden.npz"))
    x = modelzoo.synthetic_input(batch)
    _, G = _build("resnet50", batch, "int8")
    net = _run(G, "int8", x)
    logits, info = net.read_tensor("fc1000")
    logits = _valid(logits, info).reshape(batch, -1)
    # every image of the batch against the committed oracle logits (32 goldens: 16 different winning classes)
    np.testing.assert_array_equal(logits, gold["logits_int8"][:batch])
    assert (net.get_output().argmax(1) == gold["top1_int8"][:batch]).all()
    assert len(set(gold["top1_int8"][:batch].tolist())) >= 4
    _, G4 = _build("resnet50", 4, "int8")
    net4 = _run(G4, "int8", x[4:8])
    l4, i4 = net4.read_tensor("fc1000")
    np.testing.assert_array_equal(logits[4:8], _valid(l4, i4).reshape(4, -1))
    if batch > 8:   # a permuted batch permutes the result
        perm = np.random.default_rng(0).permutation(batch)
        netp = _run(G, "int8", x[perm])
        lp, ip = netp.read_tensor("fc1000")
        np.testing.assert_array_equal(_valid(lp, ip).reshape(batch, -1), logits[perm])
    prob = net.get_output()
    np.testing.assert_allclose(prob.sum(1), 1.0, rtol=1e-5)


@pytest.mark.parametrize("batch", [1, 8])
def test_resnet50_fp32_golden(batch):
    """C1 (batch 1) and a full batch: fp32 logits of every image against the fp32 oracle's."""
    from anakin_b200 import modelzoo
    from oracle import pyoracle as O
    gold = np.load(os.path.join(GOLD, "resnet50_golden.npz"))
    g, G = _build("resnet50", batch, "fp32")
    net = _run(G, "fp32", modelzoo.synthetic_input(batch))
    _check_fp32_logits(O, gold["logits_fp32"][:batch], _logits(net, "fc1000", batch), "resnet50 fp32 b%d" % batch,
                       gold["logit_offset"])
    got = net.get_output()
    mr, md = O.tensor_cmp(gold["prob_fp32"][:batch], got)
    assert md < 1e-3 or mr <= 1e-3, (mr, md)
    assert (got.argmax(1) == gold["top1_fp32"][:batch]).all()


def test_graph_save_reload_runs_identically():
    """Graph::save of the optimised graph reloads and runs (net_exec_test.cpp:107 flow)."""
    from anakin_b200 import api, modelzoo
    g, G = _build("tiny_resnet", 2, "int8")
    x = modelzoo.synthetic_input(2, 32)
    a = _run(G, "int8", x).get_output()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "opt.anakin.bin")
        G.save(p)
        G2 = api.Graph.from_file(p)
        G2.Optimize()
        b = _run(G2, "int8", x).get_output()
    np.testing.assert_array_equal(a, b)


def test_eager_equals_cuda_graph():
    from anakin_b200 import modelzoo
    g, G = _build("tiny_resnet", 2, "int8")
    x = modelzoo.synthetic_input(2, 32)
    a = _run(G, "int8", x, graph=False)
    a.prediction(); a.sync()
    assert not a.cuda_graph_active()
    b = _run(G, "int8", x, graph=True)
    b.prediction(); b.sync()
    assert b.cuda_graph_active()
    np.testing.assert_array_equal(a.get_output(), b.get_output())


def test_resnet101_int8_golden():
    """BASELINE config C4 model (per-GPU shard of 4 images)."""
    from anakin_b200 import modelzoo
    gold = np.load(os.path.join(GOLD, "resnet101_golden.npz"))
    g, G = _build("resnet101", 4, "int8")
    net = _run(G, "int8", modelzoo.synthetic_input(4))
    got = net.get_output()
    assert (got.argmax(1) == gold["top1_int8"][:4]).all()
    logits, info = net.read_tensor("fc1000")
    np.testing.assert_array_equal(_valid(logits, info).reshape(4, -1), gold["logits_int8"][:4])


def test_mobilenet_v1_int8_golden(oracle):
    """MobileNet-v1 in INT8 at the batch size C5 names: 13 INT8 depthwise layers + 13 1x1 layers + the 3x3/s2 stem; logits
    and top-1 against the committed oracle outputs, two depthwise edges against a fresh oracle run."""
    from anakin_b200 import modelzoo
    from oracle import model_walker as W
    gold = np.load(os.path.join(GOLD, "mobilenet_v1_golden.npz"))
    batch = 16
    g, G = _build("mobilenet_v1", batch, "int8")
    x = modelzoo.synthetic_input(batch)
    net = _run(G, "int8", x)
    got = net.get_output()
    np.testing.assert_array_equal(_logits(net, "fc7", batch), gold["logits_int8"])
    assert (got.argmax(1) == gold["top1_int8"]).all() and len(set(gold["top1_int8"].tolist())) >= 3
    scales = {k: float(np.float32(v)) for k, v in modelzoo.load_calibration("mobilenet_v1").items()}
    g2 = modelzoo.build("mobilenet_v1", batch=2, precision="int8")
    _, trace = W.run_int8(g2, x[:2], scales, return_intermediate=True)
    for node in ("conv1", "conv2_dw", "conv3_dw", "conv7_sep", "conv14_dw", "conv14_sep"):
        arr, info = net.read_tensor(node)
        want_t = trace[node][0]
        np.testing.assert_array_equal(_valid(arr, info)[:2].reshape(want_t.shape), want_t, err_msg=node)


def test_tiny_mobilenet_fp32_and_fp16(oracle):
    from anakin_b200 import modelzoo
    gold = np.load(os.path.join(GOLD, "tiny_mobilenet_golden.npz"))
    nb = gold["top1_fp32"].shape[0]
    x = modelzoo.synthetic_input(nb, 32)
    g, G = _build("tiny_mobilenet", nb, "fp32")
    net = _run(G, "fp32", x)
    _check_fp32_logits(oracle, gold["logits_fp32"], _logits(net, "fc7", nb), "tiny_mobilenet fp32", gold["logit_offset"])
    assert (net.get_output().argmax(1) == gold["top1_fp32"]).all()
    g, G = _build("tiny_mobilenet", nb, "fp16")
    net16 = _run(G, "fp16", x)
    l16, l32 = _logits(net16, "fc7", nb).astype(np.float32), gold["logits_fp32"]
    bound = 4.0 * np.sqrt(10.0) * 2.0 ** -11 * float(np.abs(l32 + gold["logit_offset"]).max())   # 10 fp16 edges in series
    assert np.abs(l16 - l32).max() <= bound, (float(np.abs(l16 - l32).max()), bound)


def test_vgg16_fp32_golden():
    """BASELINE config C3 model: 3x3 convs + the 25088x4096 fc (NCHW-flatten order)."""
    from anakin_b200 import modelzoo
    from oracle import pyoracle as O
    gold = np.load(os.path.join(GOLD, "vgg16_golden.npz"))
    batch = 4                                   # the batch size C3 names
    g, G = _build("vgg16", batch, "fp32")
    net = _run(G, "fp32", modelzoo.synthetic_input(batch))
    _check_fp32_logits(O, gold["logits_fp32"], _logits(net, "fc8", batch), "vgg16 fp32 b4", gold["logit_offset"])
    got = net.get_output()
    mr, md = O.tensor_cmp(gold["prob_fp32"], got)
    assert md < 1e-3 or mr <= 1e-3, (mr, md)
    assert (got.argmax(1) == gold["top1_fp32"]).all() and len(set(gold["top1_fp32"].tolist())) >= 3


def test_mobilenet_v1_fp16_vs_fp32_oracle():
    """BASELINE config C5 model: depthwise + 1x1 path in FP16. The reference has no FP16 NV kernels
    (every AK_HALF impl is SaberUnImplError), so the oracle is the fp32 CPU result with an fp16-sized
    tolerance on the probabilities; FP32 through the same graph must meet the 1e-3 criterion."""
    from anakin_b200 import modelzoo
    from oracle import pyoracle as O
    gold = np.load(os.path.join(GOLD, "mobilenet_v1_golden.npz"))
    batch = 16                                  # the batch size C5 names
    x = modelzoo.synthetic_input(batch)
    g, G = _build("mobilenet_v1", batch, "fp32")
    net32 = _run(G, "fp32", x)
    _check_fp32_logits(O, gold["logits_fp32"], _logits(net32, "fc7", batch), "mobilenet fp32 b16", gold["logit_offset"])
    g, G = _build("mobilenet_v1", batch, "fp16")
    net16 = _run(G, "fp16", x)
    got16 = net16.get_output()
    assert np.isfinite(got16).all()
    # FP16 storage between the 28 layers: every edge tensor is rounded to 11 significant bits (relative 2^-11 each).
    # Derived bound on a logit, errors taken as independent over the L = 28 roundings in series:
    #   |dlogit| <= 4 * sqrt(L) * 2^-11 * max|logit|   (4 sigma), i.e. 1.04e-2 of the logit scale
    l16, l32 = _logits(net16, "fc7", batch).astype(np.float32), gold["logits_fp32"]
    bound = 4.0 * np.sqrt(28.0) * 2.0 ** -11 * float(np.abs(l32 + gold["logit_offset"]).max())
    assert np.abs(l16 - l32).max() <= bound, (float(np.abs(l16 - l32).max()), bound)
    # top-1 must agree wherever the fp32 margin is larger than twice that bound
    srt = np.sort(l32, axis=1)
    clear = (srt[:, -1] - srt[:, -2]) > 2 * bound
    assert clear.sum() >= 2, int(clear.sum())     # the random net's margins are small: only some images decide clearly
    assert (got16.argmax(1)[clear] == gold["top1_fp32"][clear]).all()


def test_cpp_example_program_runs():
    """examples/example_nv_cnn_net.cpp (the reference's user program) end to end in C++."""
    import subprocess
    from anakin_b200 import modelzoo
    from test_cpu_host import _build_example
    gold = np.load(os.path.join(GOLD, "tiny_resnet_golden.npz"))
    with tempfile.TemporaryDirectory() as d:
        exe = _build_example(d)
        model = os.path.join(d, "tiny.anakin.bin")
        modelzoo.save(modelzoo.build("tiny_resnet", 1, "int8"), model)
        r = subprocess.run([exe, model, "2", "int8"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    assert "aveage time" in r.stdout and r.stdout.count("top-1 class") == 2, r.stdout


def test_worker_sync_prediction_two_threads():
    """Worker<NV,INT8>(model, 2): per-thread Nets built from one loaded graph (worker.cpp:10-151)."""
    from anakin_b200 import api, modelzoo
    gold = np.load(os.path.join(GOLD, "tiny_resnet_golden.npz"))
    with tempfile.TemporaryDirectory() as d:
        model = os.path.join(d, "tiny.anakin.bin")
        modelzoo.save(modelzoo.build("tiny_resnet", 4, "int8"), model)
        w = api.Worker(model, "int8", threads=2, devices=(0,), batch=4)
        x = modelzoo.synthetic_input(4, 32)
        for _ in range(6):
            out = w.sync_prediction(x, 4 * 12).reshape(4, 12)[:, :10]
            np.testing.assert_allclose(out, gold["prob_int8"][:4], rtol=1e-4, atol=1e-6)
        del w


def test_worker_async_prediction_pipelined_matches_single_net():
    """Worker::async_prediction / async_get_result (worker.h:77-92) on pinned buffers, 3 threads, requests with
    distinct inputs in flight: every result equals what one Net computes for that input, in submission order."""
    import torch
    from anakin_b200 import anakin_bin, api, modelzoo
    batch, nreq = 4, 12
    g = modelzoo.build("tiny_resnet", batch, "int8")
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    net = api.Net(G, "int8")
    xs = [modelzoo.synthetic_input(batch, 32, seed=100 + i) for i in range(nreq)]
    want = []
    for x in xs:
        net.set_input("input_0", x)
        net.prediction()
        want.append(net.get_output().copy())
    with tempfile.TemporaryDirectory() as d:
        model = os.path.join(d, "tiny.anakin.bin")
        modelzoo.save(g, model)
        w = api.Worker(model, "int8", threads=3, devices=(0,), batch=batch)
        w.wait_ready()
        out_count = want[0].size // want[0].shape[1] * 12      # rows are stored with 12 (padded) floats
        ins = [torch.from_numpy(x).pin_memory() for x in xs]
        outs = [torch.zeros(out_count, dtype=torch.float32).pin_memory() for _ in range(nreq)]
        inflight = 0
        for i in range(nreq):
            if inflight == 6:
                w.async_get_result()
                inflight -= 1
            w.async_prediction_ptr(ins[i].data_ptr(), ins[i].numel(), outs[i].data_ptr(), outs[i].numel())
            inflight += 1
        while inflight:
            w.async_get_result()
            inflight -= 1
        for i in range(nreq):
            got = outs[i].numpy().reshape(batch, 12)[:, :want[i].shape[1]]
            np.testing.assert_array_equal(got, want[i])
        assert any((want[0] != want[i]).any() for i in range(1, nreq)), "inputs must differ for the order check"
        # a request one element short or long fails alone, as Net.set_input would; the one queued after it is served
        for n in (ins[0].numel() - 1, ins[0].numel() + 1):
            outs[1].zero_()
            w.async_prediction_ptr(ins[0].data_ptr(), n, outs[0].data_ptr(), outs[0].numel())
            w.async_prediction_ptr(ins[1].data_ptr(), ins[1].numel(), outs[1].data_ptr(), outs[1].numel())
            with pytest.raises(api.AnakinError, match="input element count does not match the input tensor"):
                w.async_get_result()
            w.async_get_result()
            np.testing.assert_array_equal(outs[1].numpy().reshape(batch, 12)[:, :want[1].shape[1]], want[1])
        del w


def test_activation_sharing_and_weight_arena():
    """MemoryScheduler-style edge buffer sharing (memory_scheduler.cpp, net.cpp:812-898) must not change results and
    must shrink the footprint; two Nets of one Graph on one device share every packed weight image
    (graph_global_mem.h:78-250, worker.cpp:10-53)."""
    from anakin_b200 import api, modelzoo
    batch = 2
    gold = np.load(os.path.join(GOLD, "resnet50_golden.npz"))
    g, G = _build("resnet50", batch, "int8")
    x = modelzoo.synthetic_input(batch)
    b0, e0, h0, m0 = api.weight_arena_stats()
    keep = _run(G, "int8", x, keep_edges=True)
    b1, e1, h1, m1 = api.weight_arena_stats()
    shared = _run(G, "int8", x, keep_edges=False)
    b2, e2, h2, m2 = api.weight_arena_stats()
    # same answers with shared buffers, over graph replays too
    want = keep.get_output()
    np.testing.assert_array_equal(shared.get_output(), want)
    shared.prediction(); shared.prediction(); shared.sync()
    np.testing.assert_array_equal(shared.get_output(), want)
    assert (want.argmax(1) == gold["top1_int8"][:batch]).all()
    # footprint: >= 3.5x smaller than one buffer per edge (the largest edge of all -- conv1's 112 x 112 output -- no
    # longer exists at all: the stem kernel pools it in shared memory; with it the ratio was > 4)
    assert shared.activation_bytes_unshared() == keep.activation_bytes()
    assert shared.activation_bytes() * 3.5 <= shared.activation_bytes_unshared(), (
        shared.activation_bytes(), shared.activation_bytes_unshared())
    # weights: the second Net built nothing new and points at the first Net's device images
    n_w = len(keep.weight_ptrs())
    assert n_w >= 54 and m1 - m0 == n_w and e1 - e0 == n_w
    assert m2 == m1 and e2 == e1 and b2 == b1 and h2 - h1 == n_w
    assert keep.weight_ptrs() == shared.weight_ptrs() and all(keep.weight_ptrs())
    del keep, shared
    import gc
    gc.collect()
    assert api.weight_arena_stats()[1] == e0      # images are freed with their last Net


def test_calibrator_maxabs_matches_the_oracle_table_and_its_table_runs_int8(oracle):
    """anakin_b200/calibrate.py (the reference's Calibrator / EntropyCalibrator, calibrator.h, entropy_calibrator.cpp) on
    the product's own FP32 GPU path: the max-abs table equals the committed oracle table (same 8 calibration images), and
    an INT8 net built from the PRODUCT's table is bit-exact against the oracle run with that same table."""
    import json
    from anakin_b200 import anakin_bin, api, calibrate, modelzoo
    from oracle import model_walker as W
    g = modelzoo.build("tiny_resnet", batch=1)
    cal_x = modelzoo.synthetic_input(8, 32, seed=1000)
    cal = calibrate.Calibrator(g, calibrate.BatchStream([cal_x[:4], cal_x[4:]]), algo="maxabs")
    table = cal.generate_calibrator_table()
    with open(os.path.join(GOLD, "tiny_resnet_calib.json")) as f:
        want = json.load(f)["edge_scales"]
    assert set(want) <= set(table), sorted(set(want) - set(table))
    for k, v in want.items():
        assert abs(table[k] - v) <= 2e-3 * v, (k, table[k], v)       # 3xTF32 GPU maxima vs the fp32 CPU oracle's
    # the table is usable end to end: INT8 net from it == oracle walker with it, bit for bit
    batch = 4
    g8 = modelzoo.apply_int8(modelzoo.build("tiny_resnet", batch=batch), table)
    G = api.Graph.from_bytes(anakin_bin.dumps(g8))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    x = modelzoo.synthetic_input(batch, 32)
    net = _run(G, "int8", x)
    scales = {k: float(np.float32(v)) for k, v in table.items()}
    ref, trace = W.run_int8(g8, x, scales, return_intermediate=True)
    logits, info = net.read_tensor("fc")
    np.testing.assert_array_equal(_valid(logits, info).reshape(batch, -1), trace["fc"][0].reshape(batch, -1))
    assert (net.get_output().argmax(1) == ref["prob_out"].argmax(1)).all()


def test_calibrator_entropy_table_is_tighter_and_usable():
    """algo='entropy': KL thresholds never exceed the max-abs scale, and the resulting INT8 net still classifies like the
    FP32 net on most images (the threshold search is exercised end to end on real activation histograms)."""
    from anakin_b200 import anakin_bin, api, calibrate, modelzoo
    g = modelzoo.build("tiny_resnet", batch=1)
    cal_x = modelzoo.synthetic_input(8, 32, seed=1000)
    stream = calibrate.BatchStream([cal_x])
    cal = calibrate.Calibrator(g, stream, algo="entropy")
    ent = cal.generate_calibrator_table()
    mx = calibrate.Calibrator(g, stream, algo="maxabs").generate_calibrator_table()
    assert ent.keys() == mx.keys()
    assert all(ent[k] <= mx[k] * (1 + 1e-6) for k in mx)
    assert any(ent[k] < 0.98 * mx[k] for k in mx)                       # some tensor is actually clipped
    assert all(129 <= t <= calibrate.BIN_NUM for t in cal.thresh_map.values())


def test_weight_arena_export_import_round_trip():
    """Multi-GPU replicas receive the packed weights by one broadcast (anakin_b200/dist.py::broadcast_weight_arena). The
    mechanism on one GPU, in a fresh process (its arena holds nothing else): export the arena of a Net, drop the Net,
    build the same Net in receive mode (buffers only -- its output is wrong), import the exported image: bit-identical."""
    _arena_round_trip("tiny_resnet", "int8")


@pytest.mark.parametrize("name,precision", [("tiny_mobilenet", "int8"), ("tiny_mobilenet", "fp16")])
def test_weight_arena_export_import_round_trip_depthwise_and_fp16(name, precision):
    """The same round trip over the other image layouts receive mode must size: depthwise images, and fp16 ones."""
    _arena_round_trip(name, precision)


def _arena_round_trip(name, precision):
    import subprocess
    import sys
    code = r'''
import gc, sys
import numpy as np, torch
sys.path.insert(0, %r)
from anakin_b200 import anakin_bin, api, modelzoo
NAME, PREC = %r, %r
def build(batch):
    G = api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build(NAME, batch=batch, precision=PREC)))
    G.ResetBatchSize("input_0", batch); G.Optimize()
    return G
def run(net, x):
    net.set_input("input_0", x); net.prediction(); net.sync(); return net.get_output().copy()
x = modelzoo.synthetic_input(3, 32)
G = build(3); a = api.Net(G, PREC, device=0)
want = run(a, x)
nbytes = api.weight_arena_flat_bytes(0)
assert nbytes > 0 and nbytes %% 256 == 0
flat = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
api.weight_arena_export(0, flat.data_ptr(), nbytes)
del a, G; gc.collect()
assert api.weight_arena_stats()[1] == 0, "arena must be empty once its Nets are gone"
api.weight_arena_set_receive(True)
G = build(3); b = api.Net(G, PREC, device=0)
api.weight_arena_set_receive(False)
assert api.weight_arena_flat_bytes(0) == nbytes
assert not np.array_equal(run(b, x), want), "receive mode must not have built any weights"
api.weight_arena_import(0, flat.data_ptr(), nbytes)
got = run(b, x)
np.testing.assert_array_equal(got, want)
print("ROUND_TRIP_OK", nbytes)
''' % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))), name, precision)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ROUND_TRIP_OK" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


def test_worker_threads_on_two_devices():
    """Worker with devices=[0, 1]: thread i drives GPU i from ONE process (per-device shared-memory opt-in, per-device
    weight arena, tensor maps encoded per device). Needs two GPUs (`gpurun --gpus 2`); skipped on a single-GPU box."""
    import torch
    from anakin_b200 import api, modelzoo
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    gold = np.load(os.path.join(GOLD, "tiny_resnet_golden.npz"))
    with tempfile.TemporaryDirectory() as d:
        model = os.path.join(d, "tiny.anakin.bin")
        modelzoo.save(modelzoo.build("tiny_resnet", 4, "int8"), model)
        w = api.Worker(model, "int8", threads=2, devices=(0, 1), batch=4)
        w.wait_ready()
        x = modelzoo.synthetic_input(4, 32)
        for _ in range(8):          # requests alternate between the two threads / devices
            out = w.sync_prediction(x, 4 * 12).reshape(4, 12)[:, :10]
            np.testing.assert_allclose(out, gold["prob_int8"][:4], rtol=1e-4, atol=1e-6)
        del w
