"""GPU: on-device resize and centre crop of 8-bit images of any size (b200_image_resize_run, the `<input>:ImageResize`
op). Every comparison is bit for bit, with deterministic seeds: the kernel against the numpy oracle
(tests/image_resize_oracle.py, pinned to the reference's resize by tests/test_cpu_image_resize.py), and a resizing Net
against the plain image Net fed the oracle-resized batch."""
import ctypes as C
import os
import tempfile
import zlib

import numpy as np
import pytest

import image_resize_oracle as O
from test_image_input_gpu import dilated_tiny_resnet, eager_launches

pytestmark = pytest.mark.gpu

MEAN = [123.675, 116.28, 103.53, 64.0]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375, 1 / 40.0]


def _images(sizes, c, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, c), dtype=np.uint8) for h, w in sizes]


# ---------------------------------------------------------------------------------------------- 1. kernel
def _kernel_sources(oh, ow):
    # identity, 2x down, 500x375 both ways, upscale, extreme aspect, one pixel, a 1280 x 960 "max size" image
    return [(oh, ow), (2 * oh, 2 * ow), (375, 500), (500, 375), (100, 150), (16, 1000), (1, 1), (1280, 960)]


@pytest.mark.parametrize("net_hw", [(224, 224), (200, 160)])
@pytest.mark.parametrize("s", [0, 256, 232])
@pytest.mark.parametrize("c", [1, 3, 4])
def test_kernel_equals_oracle(c, s, net_hw):
    import torch
    from anakin_b200 import api, saber_abi as A
    from gpu_util import ptr, stream_ptr
    lib = A.load()
    oh, ow = net_hw
    sizes = _kernel_sources(oh, ow)
    imgs = _images(sizes, c, zlib.crc32(repr((c, s, net_hw)).encode()))
    pix, hw = api.pack_images(imgs)
    table = (A.ImageResizeEntry * len(imgs))()
    off = 0
    for i, (h, w) in enumerate(sizes):
        rh, rw, top, left = O.geometry(h, w, s, oh, ow)
        table[i].offset, table[i].h, table[i].w = off, h, w
        table[i].rh, table[i].rw, table[i].top, table[i].left = rh, rw, top, left
        off += h * w * c
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = len(imgs), c, oh, ow
    src = torch.from_numpy(pix).cuda()
    tab = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).cuda()
    out = torch.full((len(imgs), oh, ow, c), 7, dtype=torch.uint8, device="cuda")
    A.check(lib.b200_image_resize_run(C.byref(d), ptr(src), ptr(tab), ptr(out), stream_ptr()), "image_resize")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for i, img in enumerate(imgs):
        want = O.image_resize_u8(img, s, oh, ow)
        assert np.array_equal(got[i], want), (sizes[i], int(np.abs(got[i].astype(int) - want).max()))
    # a row that is not a multiple of 4 pixels takes the byte-store instance
    if net_hw == (224, 224):
        d.out_w = 221
        out = torch.full((len(imgs), oh, 221, c), 7, dtype=torch.uint8, device="cuda")
        for i, (h, w) in enumerate(sizes):
            rh, rw, top, left = O.geometry(h, w, s, oh, 221)
            table[i].rh, table[i].rw, table[i].top, table[i].left = rh, rw, top, left
        tab = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).cuda()
        A.check(lib.b200_image_resize_run(C.byref(d), ptr(src), ptr(tab), ptr(out), stream_ptr()), "image_resize")
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        for i, img in enumerate(imgs):
            assert np.array_equal(got[i], O.image_resize_u8(img, s, oh, 221)), sizes[i]


# ---------------------------------------------------------------------------------------------- 2. Net
def _graphs(g_dict, batch, max_hw, resize_short):
    """(plain image Graph, resizing image Graph) from one model dict."""
    from anakin_b200 import anakin_bin, api
    blob = anakin_bin.dumps(g_dict)
    Gp, Gr = api.Graph.from_bytes(blob), api.Graph.from_bytes(blob)
    c = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"][1]
    for G in (Gp, Gr):
        G.set_input_image("input_0", MEAN[:c], SCALE[:c], [2, 1, 0][:c] if c == 3 else list(range(c)))
    Gr.set_input_image_resize("input_0", max_hw[0], max_hw[1], resize_short)
    for G in (Gp, Gr):
        G.ResetBatchSize("input_0", batch)
        G.Optimize()
    return Gp, Gr


def compare_nets(model, precision, batch, resize_short, size_sets, max_hw, g_dict=None, check_graph=False):
    """A resizing Net and the plain image Net fed the oracle-resized batch: same outputs bit for bit, and the resizing
    Net's input tensor holds the oracle's bytes, for every request in size_sets (one list of (h, w) per request)."""
    from anakin_b200 import api, modelzoo, saber_abi
    if g_dict is None:
        g_dict = modelzoo.build(model, batch=batch, precision=precision)
    shape = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"]
    c, H, W = shape[1], shape[2], shape[3]
    Gp, Gr = _graphs(g_dict, batch, max_hw, resize_short)
    np_, nr = api.Net(Gp, precision), api.Net(Gr, precision)
    assert nr.launched_ops() == np_.launched_ops() + 1
    assert nr.exec_order()[0] == ["input_0", "ImageResize"]
    assert [o for o in nr.exec_order()[1:]] == np_.exec_order()
    info = nr.tensor_info("input_0")
    assert (info["dtype"], info["layout"], info["c_stored"], info["bytes"]) == (7, 9, c, batch * H * W * c), info
    lib = saber_abi.load()
    for it, sizes in enumerate(size_sets):
        assert len(sizes) == batch
        imgs = _images(sizes, c, seed=1000 * it + batch)
        want_in = O.resize_batch(imgs, resize_short, H, W)
        np_.set_input_image("input_0", want_in)
        nr.set_input_images("input_0", imgs)
        n0 = lib.b200_launch_count()
        nr.prediction()
        n1 = lib.b200_launch_count()
        np_.prediction()
        n2 = lib.b200_launch_count()
        np_.sync(); nr.sync()
        if it == 0:     # eager: the resize is exactly one launch more than the plain image Net makes
            assert n1 - n0 == n2 - n1 + 1, (n1 - n0, n2 - n1)
        if check_graph and it >= 1:     # captured at the second request, replayed from the third on
            assert nr.cuda_graph_active(), it
            if it >= 2:
                assert n1 == n0, (it, n1 - n0)
        got_in = nr.read_tensor("input_0")[0]
        assert np.array_equal(got_in, want_in), (model, precision, it)
        for name in np_.out_names:
            a, b = np_.get_output(name), nr.get_output(name)
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (model, precision, name, it)
    assert nr.cuda_graph_active()
    return nr


TINY_SETS = [[(32, 32), (75, 41)], [(1, 1), (80, 96)], [(33, 64), (96, 17)]]


@pytest.mark.parametrize("precision", ["fp32", "fp16", "int8"])
@pytest.mark.parametrize("model", ["tiny_resnet", "tiny_mobilenet"])
def test_tiny_nets_resize_bit_exact(model, precision):
    compare_nets(model, precision, 2, 36, TINY_SETS, (96, 96))


def test_tiny_net_stretch_bit_exact():
    compare_nets("tiny_resnet", "int8", 2, 0, TINY_SETS, (96, 96))


BIG = [(375, 500), (500, 375), (480, 640), (960, 1280), (224, 224), (100, 150), (333, 517), (1280, 1280)]


@pytest.mark.parametrize("model,precision,batch", [("resnet50", "int8", 8), ("mobilenet_v1", "fp16", 16)])
def test_benchmark_nets_resize_bit_exact(model, precision, batch):
    sets = [(BIG * 2)[:batch], (BIG[::-1] * 2)[:batch]]
    compare_nets(model, precision, batch, 256, sets, (1280, 1280))


def test_cuda_graph_serves_requests_of_different_sizes():
    sets = [[(32, 32), (75, 41)], [(1, 1), (80, 96)], [(33, 64), (96, 17)], [(96, 96), (50, 50)], [(17, 90), (64, 33)]]
    compare_nets("tiny_resnet", "int8", 2, 40, sets, (96, 96), check_graph=True)


def test_transform_path_without_fused_stem():
    """A first conv the fused stem refuses: the image input takes the NHWC transform and the R x S plan, two launches
    more than the stem-fused twin's single one; the resized bytes feed it unchanged."""
    for precision in ("fp32", "fp16", "int8"):
        nr = compare_nets(None, precision, 2, 36, TINY_SETS, (96, 96), g_dict=dilated_tiny_resnet(2, precision))
        twin = compare_nets("tiny_resnet", precision, 2, 36, TINY_SETS, (96, 96))
        assert eager_launches(nr) == eager_launches(twin) + 2, precision


def test_net_rejections():
    from anakin_b200 import api, modelzoo
    g = modelzoo.build("tiny_resnet", 2)
    Gp, Gr = _graphs(g, 2, (96, 96), 36)
    np_, nr = api.Net(Gp, "fp32"), api.Net(Gr, "fp32")
    imgs = _images([(40, 50), (60, 70)], 3, 1)
    with pytest.raises(api.AnakinError, match="1 images, the batch is 2"):
        nr.set_input_images("input_0", imgs[:1])
    with pytest.raises(api.AnakinError, match="outside 1..max"):
        nr.set_input_images("input_0", [imgs[0], _images([(97, 10)], 3, 2)[0]])
    with pytest.raises(api.AnakinError, match="outside 1..max"):
        nr.set_input_images("input_0", [imgs[0], _images([(10, 97)], 3, 2)[0]])
    lib = api.load()
    pix, hw = api.pack_images(imgs)
    assert lib.anakin_net_set_input_images(nr._h, b"input_0", pix.ctypes.data, pix.nbytes - 1, hw.ctypes.data, 2) != 0
    assert b"pixel bytes" in lib.anakin_last_error()
    assert lib.anakin_net_set_input_images(nr._h, b"input_0", None, pix.nbytes, hw.ctypes.data, 2) != 0
    assert lib.anakin_net_set_input_images(nr._h, b"no_input", pix.ctypes.data, pix.nbytes, hw.ctypes.data, 2) != 0
    # the forms are not mixed
    with pytest.raises(api.AnakinError, match="anakin_net_set_input_images"):
        nr.set_input_image("input_0", np.zeros((2, 32, 32, 3), np.uint8))
    with pytest.raises(api.AnakinError, match="image input"):
        nr.set_input("input_0", np.zeros((2, 3, 32, 32), np.float32))
    with pytest.raises(api.AnakinError, match="fixed-size image input"):
        np_.set_input_images("input_0", imgs)
    # resize_short must be 0 or cover the (reshaped) input, checked when the Net is built, naming the node
    _, Gbad = _graphs(g, 2, (96, 96), 31)
    with pytest.raises(api.AnakinError, match="input_0.*at least max"):
        api.Net(Gbad, "fp32")
    # a rejected request leaves the Net serving
    nr.set_input_images("input_0", imgs)
    nr.prediction(); nr.sync()
    assert np.array_equal(nr.read_tensor("input_0")[0], O.resize_batch(imgs, 36, 32, 32))


def test_worker_async_resize_requests_match_a_single_net():
    import torch
    from anakin_b200 import anakin_bin, api, modelzoo
    batch = 2
    g = modelzoo.build("tiny_resnet", batch=batch, precision="int8")
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.set_input_image("input_0", MEAN[:3], SCALE[:3], [2, 1, 0])
    G.set_input_image_resize("input_0", 96, 96, 36)
    size_sets = [[(32, 32), (75, 41)], [(1, 1), (80, 96)], [(33, 64), (96, 17)], [(96, 96), (50, 50)],
                 [(17, 90), (64, 33)], [(40, 40), (41, 39)]]
    reqs = [_images(s, 3, seed=i) for i, s in enumerate(size_sets)]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tiny_resize.anakin.bin")
        G.save(path)
        G.Optimize()
        net = api.Net(G, "int8")
        want = []
        for imgs in reqs:
            net.set_input_images("input_0", imgs)
            net.prediction(); net.sync()
            want.append(net.read_tensor(net.out_names[0])[0].reshape(-1).copy())
        w = api.Worker(path, "int8", threads=2)
        w.wait_ready()
        packed = [api.pack_images(imgs) for imgs in reqs]
        pins = [(torch.from_numpy(p).pin_memory(), torch.from_numpy(h).pin_memory()) for p, h in packed]
        # request 3 is malformed: its sizes claim one more row of its second image than its pixels hold
        bad = torch.from_numpy(packed[3][1].copy()).pin_memory()
        bad[1, 0] += 1
        outs = [torch.empty(want[0].size, dtype=torch.float32).pin_memory() for _ in reqs]
        for i, ((p, h), o) in enumerate(zip(pins, outs)):
            w.async_prediction_images_ptr(p.data_ptr(), p.numel(), (bad if i == 3 else h).data_ptr(), h.shape[0],
                                          o.data_ptr(), o.numel())
        for i in range(len(reqs)):
            if i == 3:
                with pytest.raises(api.AnakinError, match="pixel bytes"):
                    w.async_get_result()
            else:
                w.async_get_result()
        for i, (o, ref) in enumerate(zip(outs, want)):
            if i != 3:
                assert np.array_equal(o.numpy(), ref), i
        got = w.sync_prediction_images(reqs[3], want[3].size)
        assert np.array_equal(got, want[3])
        with pytest.raises(api.AnakinError, match="_prediction_images"):
            w.sync_prediction_image(np.zeros((batch, 32, 32, 3), np.uint8), want[0].size)
        with pytest.raises(api.AnakinError, match="image input"):
            w.sync_prediction(np.zeros((batch, 3, 32, 32), np.float32), want[0].size)
        del w
