"""GPU: server-side batching in the Worker (Worker(..., max_delay_us=...)). The feature rests on per-image independence:
a request's rows must not depend on the slots it was given or on what the other slots hold. So every check is bit for
bit: each request's rows of graph output 0 and of the export equal the rows of the same images run through a plain Net
of that batch, where they sit in slots 0..k-1 and the other slots hold different images."""
import os
import tempfile
import threading

import numpy as np
import pytest

from test_image_resize_gpu import MEAN, SCALE, _images

pytestmark = pytest.mark.gpu

NREQ = 40


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _rows(net, export, batch):
    """(graph output 0 as stored, the export) of a Net's last prediction, one row per slot."""
    out, _ = net.read_tensor(net.out_names[0])
    return out.reshape(batch, -1).copy(), net.get_export(export, nchw=True).reshape(batch, -1).copy()


def _serve(w, reqs, submit, out_floats, clients=4):
    """Sends the requests from `clients` threads, each queueing its share as async view requests before collecting as
    many results (results come back in the Worker's submission order, so a thread may collect another's); returns every
    request's out buffer once all have completed."""
    import torch
    outs = [torch.zeros(out_floats * k, dtype=torch.float32).pin_memory() for k, _ in reqs]
    errors = []

    def client(ids):
        try:
            for i in ids:
                submit(w, reqs[i][1], outs[i])
            for _ in ids:
                w.async_get_result()
        except Exception as e:   # reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=client, args=(list(range(c, len(reqs), clients)),)) for c in range(clients)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    return [o.numpy() for o in outs]


def _check_rows(reqs, outs, want, out0, batch):
    """want(i) = (output 0 rows, export rows) of request i from the plain Net; the view holds output 0's k rows, then
    the export's."""
    for i, ((k, _), got) in enumerate(zip(reqs, outs)):
        w0, wx = want(i)
        assert _same_bits(got[:k * out0], w0[:k].reshape(-1)), ("output 0", i, k)
        assert _same_bits(got[k * out0:], wx[:k].reshape(-1)), ("export", i, k)


def _sizes(batch, seed):
    rng = np.random.default_rng(seed)
    return [int(k) for k in rng.integers(1, batch + 1, NREQ)]


# ---------------------------------------------------------------------------------------------- 1. fp32 requests
@pytest.mark.parametrize("model,precision,batch,hw,export", [
    ("resnet50", "int8", 8, 224, "pool5"),
    ("tiny_resnet", "fp32", 4, 32, "pool5"),
    ("tiny_resnet", "fp16", 4, 32, "pool5"),
    ("tiny_mobilenet", "fp32", 4, 32, "conv5_sep"),
    ("tiny_mobilenet", "fp16", 4, 32, "conv5_sep"),
])
def test_rows_equal_a_plain_net(model, precision, batch, hw, export):
    import torch
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build(model, batch=batch, precision=precision)
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    net = api.Net(G, precision, exports=[export])
    sizes = _sizes(batch, seed=len(model) + batch)
    pool = modelzoo.synthetic_input(sum(sizes), hw, seed=1000)
    filler = modelzoo.synthetic_input(batch, hw, seed=9000)
    starts = np.cumsum([0] + sizes)
    reqs = [(k, torch.from_numpy(pool[s:s + k].copy()).pin_memory()) for k, s in zip(sizes, starts)]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m.anakin.bin")
        modelzoo.save(g, path)
        w = api.Worker(path, precision, threads=3, devices=(0,), batch=batch, exports=[export], max_delay_us=200)
        sz = w.image_sizes()
        assert sz["batch"] == batch and sz["input"] == 3 * hw * hw
        out0 = sz["output"] - net.export_info(export)[1] * np.prod(net.export_info(export)[2:])
        outs = _serve(w, reqs, lambda w, x, o: w.async_prediction_ptr(x.data_ptr(), x.numel(), o.data_ptr(),
                                                                      o.numel()), sz["output"])
        # a sync request returns graph output 0's k rows
        k0, x0 = reqs[0]
        got_sync = w.sync_prediction(x0.numpy(), k0 * out0)
        del w

    def want(i):
        k, x = reqs[i]
        batch_in = filler.copy()
        batch_in[:k] = x.numpy()
        net.set_input("input_0", batch_in)
        net.prediction()
        net.sync()
        return _rows(net, export, batch)

    _check_rows(reqs, outs, want, out0, batch)
    assert _same_bits(got_sync, want(0)[0][:k0].reshape(-1))


# ---------------------------------------------------------------------------------------------- 2. image requests
def _image_graph(batch, resize=None):
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build("tiny_resnet", batch=batch, precision="int8")
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.set_input_image("input_0", MEAN[:3], SCALE[:3], [2, 1, 0])
    if resize:
        G.set_input_image_resize("input_0", 96, 96, 36, filter=resize)
    G.ResetBatchSize("input_0", batch)
    return G


def test_image_requests_equal_a_plain_net():
    import torch
    from anakin_b200 import api
    batch = 4
    G = _image_graph(batch)
    rng = np.random.default_rng(5)
    sizes = _sizes(batch, seed=5)
    reqs = [(k, torch.from_numpy(rng.integers(0, 256, (k, 32, 32, 3), dtype=np.uint8)).pin_memory()) for k in sizes]
    filler = rng.integers(0, 256, (batch, 32, 32, 3), dtype=np.uint8)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "img.anakin.bin")
        G.save(path)
        G.Optimize()
        net = api.Net(G, "int8", exports=["pool5"])
        w = api.Worker(path, "int8", threads=2, devices=(0,), exports=["pool5"], max_delay_us=200)
        sz = w.image_sizes()
        assert sz["input"] == 32 * 32 * 3
        outs = _serve(w, reqs, lambda w, x, o: w.async_prediction_image_ptr(x.data_ptr(), x.numel(), o.data_ptr(),
                                                                            o.numel()), sz["output"])
        del w

    def want(i):
        k, x = reqs[i]
        imgs = filler.copy()
        imgs[:k] = x.numpy()
        net.set_input_image("input_0", imgs)
        net.prediction()
        net.sync()
        return _rows(net, "pool5", batch)

    out0 = sz["output"] - net.export_info("pool5")[1]
    _check_rows(reqs, outs, want, out0, batch)


@pytest.mark.parametrize("resize", ["reference", "pil"])
def test_resize_requests_equal_a_plain_net(resize):
    import torch
    from anakin_b200 import api
    batch = 4
    G = _image_graph(batch, resize)
    rng = np.random.default_rng(11)
    sizes = _sizes(batch, seed=11)
    src = [(32, 32), (75, 41), (1, 1), (80, 96), (33, 64), (96, 17), (96, 96), (50, 50), (17, 90), (41, 39)]
    reqs = []
    for i, k in enumerate(sizes):
        imgs = _images([src[j] for j in rng.integers(0, len(src), k)], 3, seed=100 + i)
        pix, hw = api.pack_images(imgs)
        reqs.append((k, (imgs, torch.from_numpy(pix).pin_memory(), torch.from_numpy(hw).pin_memory())))
    filler = _images([(64, 48), (40, 90), (96, 33), (20, 20)], 3, seed=7)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "resize.anakin.bin")
        G.save(path)
        G.Optimize()
        net = api.Net(G, "int8", exports=["pool5"])
        w = api.Worker(path, "int8", threads=2, devices=(0,), exports=["pool5"], max_delay_us=200)
        sz = w.image_sizes()

        def submit(w, r, o):
            _, pix, hw = r
            w.async_prediction_images_ptr(pix.data_ptr(), pix.numel(), hw.data_ptr(), hw.shape[0], o.data_ptr(),
                                          o.numel())

        outs = _serve(w, reqs, submit, sz["output"])
        del w

    def want(i):
        k, (imgs, _, _) = reqs[i]
        net.set_input_images("input_0", list(imgs) + filler[k:])
        net.prediction()
        net.sync()
        return _rows(net, "pool5", batch)

    out0 = sz["output"] - net.export_info("pool5")[1]
    _check_rows(reqs, outs, want, out0, batch)


# ---------------------------------------------------------------------------------------------- 3. failures
def _tiny_worker_files(d, batch):
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build("tiny_resnet", batch=batch, precision="int8")
    path = os.path.join(d, "tiny.anakin.bin")
    modelzoo.save(g, path)
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return path, api.Net(G, "int8", exports=["pool5"])


def test_malformed_request_fails_alone():
    import torch
    from anakin_b200 import api, modelzoo
    batch = 4
    x = modelzoo.synthetic_input(batch, 32, seed=300)
    per = 3 * 32 * 32
    with tempfile.TemporaryDirectory() as d:
        path, net = _tiny_worker_files(d, batch)
        net.set_input("input_0", x)
        net.prediction()
        net.sync()
        w0, wx = _rows(net, "pool5", batch)
        # a 0.1 s window: the four requests below are queued long before it closes, so they form one batch
        w = api.Worker(path, "int8", threads=1, devices=(0,), exports=["pool5"], max_delay_us=100000)
        sz = w.image_sizes()
        out0 = sz["output"] - wx.shape[1]
        xin = torch.from_numpy(x.reshape(-1).copy()).pin_memory()
        outs = [torch.zeros(k * sz["output"], dtype=torch.float32).pin_memory() for k in (1, 1, 2, 1)]
        # A: image 0; B: one and a half images; C: images 1..2; D: image 3 with a result buffer one float short
        w.async_prediction_ptr(xin.data_ptr(), per, outs[0].data_ptr(), outs[0].numel())
        w.async_prediction_ptr(xin.data_ptr(), per + per // 2, outs[1].data_ptr(), outs[1].numel())
        w.async_prediction_ptr(xin.data_ptr() + 4 * per, 2 * per, outs[2].data_ptr(), outs[2].numel())
        w.async_prediction_ptr(xin.data_ptr() + 12 * per, per, outs[3].data_ptr(), outs[3].numel() - 1)
        w.async_get_result()
        with pytest.raises(api.AnakinError, match="request of %d floats: not 1..4 images of %d floats each" %
                           (per + per // 2, per)):
            w.async_get_result()
        w.async_get_result()
        with pytest.raises(api.AnakinError, match="out_count %d, the result of 1 images is %d floats" %
                           (sz["output"] - 1, sz["output"])):
            w.async_get_result()
        got = [o.numpy() for o in outs]
        assert _same_bits(got[0][:out0], w0[0]) and _same_bits(got[0][out0:], wx[0])
        assert _same_bits(got[2][:2 * out0], w0[1:3].reshape(-1)) and _same_bits(got[2][2 * out0:], wx[1:3].reshape(-1))
        assert not got[1].any() and not got[3].any()
        # more images than the batch fails alone, and the Worker keeps serving
        big = modelzoo.synthetic_input(batch + 1, 32, seed=300)
        with pytest.raises(api.AnakinError, match="not 1..4 images"):
            w.sync_prediction(big, (batch + 1) * out0)
        assert _same_bits(w.sync_prediction(x[3:4], out0), w0[3])
        del w


def test_batching_off_refuses_fewer_images_than_the_batch():
    from anakin_b200 import api, modelzoo
    batch = 4
    with tempfile.TemporaryDirectory() as d:
        path, _ = _tiny_worker_files(d, batch)
        w = api.Worker(path, "int8", threads=1, devices=(0,))
        w.wait_ready()
        with pytest.raises(api.AnakinError, match="input element count does not match the input tensor"):
            w.sync_prediction(modelzoo.synthetic_input(1, 32), 10)
        del w


def test_lone_request_completes_after_the_window():
    from anakin_b200 import api, modelzoo
    batch = 4
    x = modelzoo.synthetic_input(1, 32, seed=400)
    with tempfile.TemporaryDirectory() as d:
        path, _ = _tiny_worker_files(d, batch)
        w = api.Worker(path, "int8", threads=1, devices=(0,), max_delay_us=1000)
        sz = w.image_sizes()
        got = w.sync_prediction(x, sz["output"])
        assert np.isfinite(got).all() and abs(float(got.sum()) - 1.0) < 1e-3   # one softmax row
        del w
