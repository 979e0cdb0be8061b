"""GPU: the Pillow filter of the on-device resize (b200_image_resize_pil_run, the `<input>:ImageResize` op with
image_resize_filter 1). Every comparison is bit for bit, with deterministic seeds: the kernels against the numpy
restatement (tests/pil_resize_oracle.py, pinned to Pillow by tests/test_cpu_image_resize_pil.py), and a Net with the
filter against the plain image Net fed the restated bytes."""
import ctypes as C
import os
import tempfile
import zlib

import numpy as np
import pytest

import pil_resize_oracle as P

pytestmark = pytest.mark.gpu

MEAN = [123.675, 116.28, 103.53, 64.0]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375, 1 / 40.0]


def _images(sizes, c, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, c), dtype=np.uint8) for h, w in sizes]


# ---------------------------------------------------------------------------------------------- 1. kernels
def _kernel_sources(oh, ow):
    # identity, 2x down, 500x375 both ways, upscale, extreme aspect, one pixel, a phone photo, and the pass-order
    # cases on both sides of Pillow's switch
    return ([(oh, ow), (2 * oh, 2 * ow), (375, 500), (500, 375), (100, 150), (16, 1000), (1, 1), (3024, 4032)]
            + [(h, w) for h, w, _, _ in P.PASS_ORDER_CASES[:10]])


def _run_kernel(lib, A, imgs, c, s, oh, ow, max_hw):
    import torch
    from anakin_b200 import api
    from gpu_util import ptr, stream_ptr
    pix, hw = api.pack_images(imgs)
    table = (A.ImageResizeEntry * len(imgs))()
    off = 0
    for i, img in enumerate(imgs):
        h, w = img.shape[:2]
        v = [C.c_int32() for _ in range(4)]
        A.check(lib.b200_image_resize_geometry_ex(h, w, s, oh, ow, 1, *[C.byref(x) for x in v]), "geometry_ex")
        table[i].offset, table[i].h, table[i].w = off, h, w
        table[i].rh, table[i].rw, table[i].top, table[i].left = [x.value for x in v]
        off += h * w * c
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = len(imgs), c, oh, ow
    nbytes = C.c_size_t()
    A.check(lib.b200_image_resize_pil_workspace(C.byref(d), max_hw[0], max_hw[1], s, C.byref(nbytes)), "workspace")
    ws = torch.full((nbytes.value,), 0xA5, dtype=torch.uint8, device="cuda")
    src = torch.from_numpy(pix).cuda()
    tab = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).cuda()
    out = torch.full((len(imgs), oh, ow, c), 7, dtype=torch.uint8, device="cuda")
    A.check(lib.b200_image_resize_pil_run(C.byref(d), max_hw[0], max_hw[1], s, ptr(src), ptr(tab), ptr(ws), ptr(out),
                                          stream_ptr()), "image_resize_pil")
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("net_hw", [(224, 224), (200, 160)])
@pytest.mark.parametrize("s", [0, 256, 232])
@pytest.mark.parametrize("c", [1, 2, 3, 4])
def test_kernel_equals_restatement(c, s, net_hw):
    from anakin_b200 import saber_abi as A
    lib = A.load()
    oh, ow = net_hw
    sizes = _kernel_sources(oh, ow)
    imgs = _images(sizes, c, zlib.crc32(repr((c, s, net_hw)).encode()))
    max_hw = (max(h for h, _ in sizes), max(w for _, w in sizes))
    widths = [ow] + ([221] if net_hw == (224, 224) else [])     # 221: the byte-store instance
    for w_out in widths:
        got = _run_kernel(lib, A, imgs, c, s, oh, w_out, max_hw)
        for i, img in enumerate(imgs):
            want = P.resize_u8(img, s, oh, w_out)
            assert np.array_equal(got[i], want), (sizes[i], w_out, int(np.abs(got[i].astype(int) - want).max()))


def test_kernel_on_stripes_of_a_phone_photo():
    """The 3.3-pixel stripes of the golden fixture, 12x down: the antialiased result, bit for bit."""
    from anakin_b200 import saber_abi as A
    lib = A.load()
    img = P.case_image(3024, 4032, 3, "stripes", 0)
    got = _run_kernel(lib, A, [img, img[:, :3000]], 3, 256, 224, 224, (3024, 4032))
    assert np.array_equal(got[0], P.resize_u8(img, 256, 224, 224))
    assert np.array_equal(got[1], P.resize_u8(img[:, :3000], 256, 224, 224))
    assert got[0].std() < 10


# ---------------------------------------------------------------------------------------------- 2. Net
def _graphs(g_dict, batch, max_hw, resize_short, filt="pil"):
    """(plain image Graph, resizing image Graph with `filt`) from one model dict."""
    from anakin_b200 import anakin_bin, api
    blob = anakin_bin.dumps(g_dict)
    Gp, Gr = api.Graph.from_bytes(blob), api.Graph.from_bytes(blob)
    c = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"][1]
    for G in (Gp, Gr):
        G.set_input_image("input_0", MEAN[:c], SCALE[:c], [2, 1, 0][:c] if c == 3 else list(range(c)))
    Gr.set_input_image_resize("input_0", max_hw[0], max_hw[1], resize_short, filter=filt)
    for G in (Gp, Gr):
        G.ResetBatchSize("input_0", batch)
        G.Optimize()
    return Gp, Gr


def compare_nets(model, precision, batch, resize_short, size_sets, max_hw, check_graph=False):
    """A Net with the Pillow filter and the plain image Net fed the restated batch: same outputs bit for bit, and the
    resizing Net's input tensor holds the restated bytes, for every request in size_sets."""
    from anakin_b200 import api, modelzoo, saber_abi
    g_dict = modelzoo.build(model, batch=batch, precision=precision)
    shape = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"]
    c, H, W = shape[1], shape[2], shape[3]
    Gp, Gr = _graphs(g_dict, batch, max_hw, resize_short)
    np_, nr = api.Net(Gp, precision), api.Net(Gr, precision)
    assert nr.launched_ops() == np_.launched_ops() + 1
    assert nr.exec_order()[0] == ["input_0", "ImageResize"]
    assert nr.exec_order()[1:] == np_.exec_order()
    lib = saber_abi.load()
    for it, sizes in enumerate(size_sets):
        imgs = _images(sizes, c, seed=1000 * it + batch)
        want_in = P.resize_batch(imgs, resize_short, H, W)
        np_.set_input_image("input_0", want_in)
        nr.set_input_images("input_0", imgs)
        n0 = lib.b200_launch_count()
        nr.prediction()
        n1 = lib.b200_launch_count()
        np_.prediction()
        n2 = lib.b200_launch_count()
        np_.sync(); nr.sync()
        if it == 0:     # eager: taps, first pass, second pass
            assert n1 - n0 == n2 - n1 + 3, (n1 - n0, n2 - n1)
        if check_graph and it >= 2:
            assert nr.cuda_graph_active() and n1 == n0, (it, n1 - n0)
        assert np.array_equal(nr.read_tensor("input_0")[0], want_in), (model, precision, it)
        for name in np_.out_names:
            a, b = np_.get_output(name), nr.get_output(name)
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (model, precision, name, it)
    assert nr.cuda_graph_active()
    return nr


TINY_SETS = [[(32, 32), (75, 41)], [(1, 1), (80, 96)], [(33, 64), (96, 17)]]


@pytest.mark.parametrize("precision", ["fp32", "fp16", "int8"])
@pytest.mark.parametrize("model", ["tiny_resnet", "tiny_mobilenet"])
def test_tiny_nets_pil_resize_bit_exact(model, precision):
    compare_nets(model, precision, 2, 36, TINY_SETS, (96, 96))


def test_tiny_net_pil_stretch_bit_exact():
    compare_nets("tiny_resnet", "int8", 2, 0, TINY_SETS + [[(3000, 16), (16, 40)]], (3000, 96))


BIG = [(375, 500), (500, 375), (480, 640), (960, 1280), (224, 224), (100, 150), (333, 517), (3024, 4032)]


@pytest.mark.parametrize("model,precision,batch", [("resnet50", "int8", 8), ("mobilenet_v1", "fp16", 16)])
def test_benchmark_nets_pil_resize_bit_exact(model, precision, batch):
    sets = [(BIG * 2)[:batch], (BIG[::-1] * 2)[:batch]]
    compare_nets(model, precision, batch, 256, sets, (3024, 4032))


def test_cuda_graph_serves_requests_of_different_tap_counts():
    """Upscales (3 taps) to 16x downscales (35 taps), on one captured graph."""
    sets = [[(32, 32), (75, 41)], [(600, 600), (1, 1)], [(40, 600), (600, 41)], [(96, 96), (590, 5)],
            [(17, 90), (64, 33)], [(600, 300), (300, 600)]]
    compare_nets("tiny_resnet", "int8", 2, 36, sets, (600, 600), check_graph=True)


def test_filter_zero_equals_no_attribute():
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build("tiny_resnet", batch=2, precision="int8")
    blob = anakin_bin.dumps(g)
    nets = []
    for explicit in (False, True):
        G = api.Graph.from_bytes(blob)
        G.set_input_image("input_0", MEAN[:3], SCALE[:3], [2, 1, 0])
        G.set_input_image_resize("input_0", 96, 96, 36)
        if explicit:
            assert api.load().anakin_graph_set_input_image_resize_filter(G._h, b"input_0", 0) == 0
        else:       # no image_resize_filter attribute at all
            with tempfile.TemporaryDirectory() as d:
                p = os.path.join(d, "m.anakin.bin")
                G.save(p)
                with open(p, "rb") as f:
                    gd = anakin_bin.loads(f.read())
            gd["nodes"][[n["op"] for n in gd["nodes"]].index("Input")]["attrs"].pop("image_resize_filter", None)
            G = api.Graph.from_bytes(anakin_bin.dumps(gd))
        G.Optimize()
        nets.append(api.Net(G, "int8"))
    for it, sizes in enumerate(TINY_SETS):
        imgs = _images(sizes, 3, seed=it)
        outs = []
        for n in nets:
            n.set_input_images("input_0", imgs)
            n.prediction(); n.sync()
            outs.append((n.read_tensor("input_0")[0], n.get_output(n.out_names[0])))
        assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1]), it


def test_net_rejects_a_malformed_filter_attribute():
    from anakin_b200 import anakin_bin, api, modelzoo
    Gp, Gr = _graphs(modelzoo.build("tiny_resnet", 2), 2, (96, 96), 36)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        Gr.save(p)
        with open(p, "rb") as f:
            gd = anakin_bin.loads(f.read())
    gd["nodes"][[n["op"] for n in gd["nodes"]].index("Input")]["attrs"]["image_resize_filter"] = 2
    G = api.Graph.from_bytes(anakin_bin.dumps(gd))
    with pytest.raises(api.AnakinError, match="malformed image resize attributes on Input input_0"):
        api.Net(G, "fp32")


def test_worker_async_pil_requests_match_a_single_net():
    import torch
    from anakin_b200 import anakin_bin, api, modelzoo
    batch = 2
    g = modelzoo.build("tiny_resnet", batch=batch, precision="int8")
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.set_input_image("input_0", MEAN[:3], SCALE[:3], [2, 1, 0])
    G.set_input_image_resize("input_0", 600, 600, 36, filter="pil")
    size_sets = [[(32, 32), (75, 41)], [(1, 1), (600, 96)], [(33, 64), (96, 17)], [(600, 600), (50, 50)],
                 [(590, 5), (64, 33)], [(40, 40), (41, 39)]]
    reqs = [_images(s, 3, seed=i) for i, s in enumerate(size_sets)]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tiny_resize_pil.anakin.bin")
        G.save(path)
        G.Optimize()
        net = api.Net(G, "int8")
        want = []
        for imgs in reqs:
            net.set_input_images("input_0", imgs)
            net.prediction(); net.sync()
            assert np.array_equal(net.read_tensor("input_0")[0], P.resize_batch(imgs, 36, 32, 32))
            want.append(net.read_tensor(net.out_names[0])[0].reshape(-1).copy())
        w = api.Worker(path, "int8", threads=2)
        w.wait_ready()
        packed = [api.pack_images(imgs) for imgs in reqs]
        pins = [(torch.from_numpy(p).pin_memory(), torch.from_numpy(h).pin_memory()) for p, h in packed]
        outs = [torch.empty(want[0].size, dtype=torch.float32).pin_memory() for _ in reqs]
        for _ in range(2):      # the second round replays each thread's captured graph
            for (p, h), o in zip(pins, outs):
                w.async_prediction_images_ptr(p.data_ptr(), p.numel(), h.data_ptr(), h.shape[0], o.data_ptr(),
                                              o.numel())
            for _ in reqs:
                w.async_get_result()
            for i, (o, ref) in enumerate(zip(outs, want)):
                assert np.array_equal(o.numpy(), ref), i
        got = w.sync_prediction_images(reqs[3], want[3].size)
        assert np.array_equal(got, want[3])
        del w
