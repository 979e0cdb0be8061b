"""INT8 calibration statistics on the GPU (b200_calib_stats_run / b200_calib_kl_run, Net(..., calib_stats=True),
anakin_b200/calibrate.py) against the host computation they replace (tests/calib_host_ref.py: edge read-back + numpy,
and calibrate.kl_threshold).

  maxima       bit for bit          histograms   equal integer arrays
  thresholds   equal to kl_threshold's; where one differs, the restatement's own KL values at the two bins agree to
               1e-12 relative (a near-tie inside float64 rounding of log2 and the KL sums)
"""
import functools

import numpy as np
import pytest

import calib_host_ref as H

pytestmark = pytest.mark.gpu

BINS = H.BIN_NUM
# model -> (batch, image size, batches); every case runs two or more batches so that accumulation is covered
CASES = {"tiny_resnet": (4, 32, 2), "tiny_mobilenet": (4, 32, 2), "resnet50": (8, 224, 2)}


def _graph(name, batch, precision="fp32"):
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build(name, batch=batch, precision=precision)
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return g, G


def _batches(name):
    from anakin_b200 import modelzoo
    batch, hw, nb = CASES[name]
    return [modelzoo.synthetic_input(batch, hw, seed=1000 + batch * b) for b in range(nb)]


def _passes(net, xs):
    """Both passes of the calibration statistics over xs: (float32 maxima, uint64 histograms)."""
    net.calib_reset()
    for p in (0, 1):
        net.calib_set_pass(p)
        for x in xs:
            net.set_input("input_0", x)
            net.prediction()
    mx, hs = net.calib_read()
    return mx, hs


@functools.lru_cache(maxsize=None)
def _case(name, cuda_graph=True):
    """GPU statistics of a calib_stats net (buffer sharing on) and the host statistics of a keep_edges twin."""
    from anakin_b200 import api
    g, G = _graph(name, CASES[name][0])
    net = api.Net(G, "fp32", calib_stats=True)
    if not cuda_graph:
        net.set_cuda_graph(False)
    xs = _batches(name)
    mx, hs = _passes(net, xs)
    assert net.cuda_graph_active() == cuda_graph
    assert net.activation_bytes() < net.activation_bytes_unshared()          # buffers are shared
    names = net.calib_names()
    padded = [n for n in names[1:] if net.tensor_info(n)["c_stored"] != net.tensor_info(n)["dims"][1]]
    ops = dict((n, o) for n, o in net.exec_order())
    del net
    twin = api.Net(G, "fp32", keep_edges=True)
    assert [n for n, _ in twin.exec_order()] == names[1:]
    hmax, hhist = H.host_stats(twin, names, xs)
    return dict(g=g, names=names, ops=ops, xs=xs, max=mx, hist=hs, hmax=hmax, hhist=hhist, padded=padded)


@functools.lru_cache(maxsize=None)
def _ref_thresholds(name):
    c = _case(name)
    live = [n for n in c["names"] if c["hmax"][n] > 0]
    return dict(zip(live, H.kl_thresholds([c["hhist"][n] for n in live])))


def _check_stats(c):
    for k, n in enumerate(c["names"]):
        want = np.float32(c["hmax"][n])
        assert c["max"][k].view(np.uint32) == want.view(np.uint32), (n, float(c["max"][k]), float(want))
        want_h = c["hhist"].get(n, np.zeros(BINS, np.int64))
        got_h = c["hist"][k].astype(np.int64)
        bad = np.flatnonzero(got_h != want_h)
        assert bad.size == 0, (n, bad[:5], got_h[bad[:5]], want_h[bad[:5]])


@pytest.mark.parametrize("name", ["tiny_resnet", "tiny_mobilenet", "resnet50"])
def test_statistics_equal_the_host_reduction(name):
    """tiny_resnet: side-stream projection shortcut, fused conv + pooling, the FC edge of 10 channels stored as 12;
    tiny_mobilenet: depthwise convolutions; ResNet-50 at batch 8. Shared buffers, captured CUDA graph."""
    c = _case(name)
    assert c["names"][0] == "input_0" and len(c["names"]) == len(c["ops"]) + 1
    if name == "tiny_resnet":
        assert c["padded"], "the padded FC edge must be observed"
        assert any(o.endswith("Pool") for o in c["ops"].values())
    if name == "tiny_mobilenet":
        assert any(n.endswith("_dw") for n in c["ops"]), "the depthwise convolutions must be observed"
    _check_stats(c)


def test_statistics_equal_the_host_reduction_without_cuda_graph():
    _check_stats(_case("tiny_resnet", cuda_graph=False))


@pytest.mark.parametrize("name", ["tiny_resnet", "tiny_mobilenet", "resnet50"])
def test_flag_is_invisible_when_off_and_costs_only_its_launches(name):
    from anakin_b200 import api, saber_abi
    _, G = _graph(name, CASES[name][0])
    plain = api.Net(G, "fp32")
    cal = api.Net(G, "fp32", calib_stats=True)
    assert cal.exec_order() == plain.exec_order()
    assert cal.activation_bytes() == plain.activation_bytes()
    names = cal.calib_names()
    assert names == ["input_0"] + [n for n, _ in plain.exec_order()]
    assert plain.calib_names() == []
    with pytest.raises(api.AnakinError, match="calibration statistics"):
        plain.calib_set_pass(1)
    assert cal.launched_ops() == plain.launched_ops() + len(names)
    assert len(cal.profile_ops(iters=1)) == len(plain.exec_order())       # the statistics launches are not timed
    # launches of one eager prediction, counted by the library
    lib = saber_abi.load()
    x = _batches(name)[0]
    counts = []
    for net in (plain, cal):
        net.set_cuda_graph(False)
        net.set_input("input_0", x)
        net.sync()
        before = lib.b200_launch_count()
        net.prediction()
        net.sync()
        counts.append(lib.b200_launch_count() - before)
    assert counts[1] == counts[0] + len(names), counts
    np.testing.assert_array_equal(cal.get_output(), plain.get_output())


# ------------------------------------------------------------------------------------------------ KL kernel
def _designed():
    """Histograms aimed at the branches of the restatement. Returns {label: int64[2048]}."""
    rng = np.random.default_rng(7)
    d = {}
    h = np.zeros(BINS, np.int64)                                 # post-ReLU: nearly all mass in bin 0
    h[0] = 50_000_000
    h[1:400] = (rng.exponential(1.0, 399) * 2000 * np.exp(-np.arange(399) / 60)).astype(np.int64)
    h[2047] = 1
    d["relu"] = h
    h = np.zeros(BINS, np.int64)                                 # a single spike: the max is the only value
    h[2047] = 123_456
    d["spike"] = h
    h = np.zeros(BINS, np.int64)                                 # a spike plus zeros
    h[0], h[2047] = 10_000, 77
    d["zeros_and_spike"] = h
    d["uniform"] = np.full(BINS, 1000, np.int64)
    h = np.zeros(BINS, np.int64)                                 # long sparse tail, outliers in the last bin
    h[:300] = (1e6 * np.exp(-np.arange(300) / 30.0)).astype(np.int64)
    h[rng.choice(np.arange(300, 2047), 25, replace=False)] = rng.integers(1, 4, 25)
    h[2047] = 3
    d["sparse_tail"] = h
    h = rng.integers(1, 500, BINS).astype(np.int64)              # runs of empty bins
    for a in (40, 200, 333, 700, 1200, 1500, 1900):
        h[a:a + int(rng.integers(20, 90))] = 0
    h[150:152] = 0
    d["empty_runs"] = h
    h = rng.integers(2_000_000, 4_000_000, BINS).astype(np.int64)   # totals above 2^31
    h[100:140] = 0
    d["big_total"] = h
    h = np.zeros(BINS, np.int64)                                 # nothing above bin 999: the tail of q is empty
    h[:1000] = rng.integers(1, 300, 1000)
    d["top_below_last_bin"] = h
    h = np.zeros(BINS, np.int64)                                 # counts above 2^40 in a few bins
    h[0], h[5], h[130], h[900], h[2047] = 1 << 41, 3 << 38, (1 << 40) + 12345, 987_654_321, 5
    d["huge_counts"] = h
    return d


def _paths(hist):
    """Which branches of _get_ref_q / _expand_to_q / _kl_divergence the candidates of `hist` reach (sampled)."""
    hist = np.asarray(hist, np.int64)
    hit = set()
    if hist.sum() > 2 ** 31:
        hit.add("total>2^31")
    total = int(hist.sum() - hist[0])
    for i in range(129, BINS - 1, 7):
        ref_p = hist[1:i + 1].copy()
        ref_p[i - 1] += total - int(hist[1:i].sum())
        coeff = np.float32(i) / np.float32(128)
        for j in range(128):
            start, end = np.float32(j * coeff), np.float32((j + 1) * coeff)
            s_c, e_f, s_f = int(np.ceil(start)), int(np.floor(end)), int(np.floor(start))
            zn = float(np.count_nonzero(ref_p[s_c:e_f] == 0))
            if ref_p[s_f] == 0:
                zn += s_c - start
                hit.add("zero_num_start")
            if e_f < i and ref_p[e_f] == 0:
                zn += end - e_f
                hit.add("zero_num_end")
            if coeff - zn <= 0:
                hit.add("dis<=0")
    for i in range(129, BINS - 1):
        # an empty last kept bin leaves q's last bin empty (tail_q == 0) while the histogram goes on
        if hist[i:].sum() == 0 and hist[i - 1] > 0:
            hit.add("tail_q<=0")
    return hit


def _kl_gpu(hists):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ptr, stream_ptr
    lib = A.load()
    h = torch.from_numpy(np.ascontiguousarray(np.stack(hists).astype(np.int64))).cuda()
    th = torch.zeros(len(hists), dtype=torch.int32, device="cuda")
    kl = torch.zeros((len(hists), BINS), dtype=torch.float64, device="cuda")
    A.check(lib.b200_calib_kl_run(ptr(h), len(hists), ptr(th), ptr(kl), stream_ptr()), "calib_kl_run")
    torch.cuda.synchronize()
    return th.cpu().numpy(), kl.cpu().numpy()


def _close(a, b, rel):
    if np.isinf(a) or np.isinf(b):
        return a == b
    return abs(a - b) <= rel * max(abs(a), abs(b))


def _check_threshold(hist, got, want, label):
    if got == want:
        return 0
    assert 129 <= got <= BINS - 2 and 129 <= want <= BINS - 2, (label, got, want)
    a, b = H.kl_at(hist, got), H.kl_at(hist, want)
    assert _close(a, b, 1e-12), "%s: threshold %d (KL %r) != %d (KL %r)" % (label, got, a, want, b)
    return 1


def test_kl_kernel_matches_kl_threshold():
    designed = _designed()
    hit = set()
    for h in designed.values():
        hit |= _paths(h)
    assert hit >= {"total>2^31", "zero_num_start", "zero_num_end", "dis<=0", "tail_q<=0"}, hit
    labels, hists, want = [], [], []
    for k, h in designed.items():
        labels.append(k)
        hists.append(h)
    want += H.kl_thresholds(hists)
    for name in ("tiny_resnet", "tiny_mobilenet", "resnet50"):
        c, ref = _case(name), _ref_thresholds(name)
        for n, t in ref.items():
            labels.append("%s/%s" % (name, n))
            hists.append(c["hhist"][n])
            want.append(t)
    got, kl = _kl_gpu(hists)
    near_ties = 0
    rng = np.random.default_rng(3)
    for k, (label, h) in enumerate(zip(labels, hists)):
        near_ties += _check_threshold(h, int(got[k]), int(want[k]), label)
        # the kernel's own KL values equal the restatement's, at the chosen bin and at a few others
        for i in {int(got[k]), int(want[k]), *rng.integers(129, BINS - 1, 2).tolist()}:
            if 129 <= i <= BINS - 2:
                assert _close(float(kl[k, i]), H.kl_at(h, i), 1e-10), (label, i, float(kl[k, i]), H.kl_at(h, i))
        assert np.isnan(kl[k, :129]).all() and np.isnan(kl[k, BINS - 1])
    assert near_ties <= max(1, len(hists) // 20), near_ties


# ------------------------------------------------------------------------------------------------ tables
def _check_table(c, ref_thresh, algo, cal, table):
    want_scales, want_thresh = H.table_from_stats(c["g"], c["ops"], c["names"], c["hmax"],
                                                  ref_thresh if algo == "entropy" else {})
    assert table.keys() == want_scales.keys()
    differ = set()
    for n in c["names"]:
        if cal.thresh_map.get(n) != want_thresh.get(n):
            differ.add(n)
            _check_threshold(c["hhist"][n], cal.thresh_map[n], want_thresh[n], n)
    for k, v in table.items():
        if not any(k in H.calibrate.fused_chains(c["g"], c["ops"]).get(n, [n]) for n in differ):
            assert v == want_scales[k], (k, v, want_scales[k])
    assert len(differ) <= 1, differ


@pytest.mark.parametrize("algo", ["maxabs", "entropy"])
@pytest.mark.parametrize("name", ["tiny_resnet", "resnet50"])
def test_calibrator_tables_equal_the_host_algorithm(name, algo):
    from anakin_b200 import calibrate
    c = _case(name)
    cal = calibrate.Calibrator(c["g"], calibrate.BatchStream(c["xs"]), algo=algo)
    table = cal.generate_calibrator_table()
    _check_table(c, _ref_thresholds(name) if algo == "entropy" else {}, algo, cal, table)


def test_entropy_table_runs_int8_bit_exact_against_the_oracle(oracle):
    from anakin_b200 import anakin_bin, api, calibrate, modelzoo
    from oracle import model_walker as W
    c = _case("tiny_resnet")
    table = calibrate.Calibrator(modelzoo.build("tiny_resnet", batch=1), calibrate.BatchStream(c["xs"]),
                                 algo="entropy").generate_calibrator_table()
    batch = 4
    g8 = modelzoo.apply_int8(modelzoo.build("tiny_resnet", batch=batch), table)
    G = api.Graph.from_bytes(anakin_bin.dumps(g8))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    x = modelzoo.synthetic_input(batch, 32)
    net = api.Net(G, "int8", keep_edges=True)
    net.set_input("input_0", x)
    net.prediction()
    net.sync()
    scales = {k: float(np.float32(v)) for k, v in table.items()}
    ref, trace = W.run_int8(g8, x, scales, return_intermediate=True)
    logits, info = net.read_tensor("fc")
    got = logits[..., :info["dims"][1]].reshape(batch, -1)
    np.testing.assert_array_equal(got, trace["fc"][0].reshape(batch, -1))
    assert (net.get_output().argmax(1) == ref["prob_out"].argmax(1)).all()


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("precision", ["fp16", "int8"])
def test_non_fp32_net_refuses_the_flag(precision):
    from anakin_b200 import api
    _, G = _graph("tiny_resnet", 2, precision)
    with pytest.raises(api.AnakinError, match="calibration statistics need an FP32 net"):
        api.Net(G, precision, calib_stats=True)


def test_image_input_refuses_the_flag():
    from anakin_b200 import anakin_bin, api, modelzoo
    G = api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build("tiny_resnet", batch=2)))
    G.set_input_image("input_0", [127.5, 127.5, 127.5], [1 / 128.0] * 3)
    G.ResetBatchSize("input_0", 2)
    G.Optimize()
    with pytest.raises(api.AnakinError, match="8-bit image input"):
        api.Net(G, "fp32", calib_stats=True)
