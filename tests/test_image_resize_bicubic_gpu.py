"""GPU: Pillow's BICUBIC filter of the on-device resize (b200_image_crop_resize_run with B200_IMAGE_RESIZE_PIL_BICUBIC,
the `<input>:ImageResize` op with image_resize_filter 3). Every comparison is bit for bit, with deterministic seeds:
the kernels against the numpy restatement (tests/pil_bicubic_oracle.py, pinned to Pillow by
tests/test_cpu_image_resize_bicubic.py) applied to each box cut out of its frame (the cvtColor image for NV12 /
I420); Nets and a batching Worker with the filter against the plain image Net fed the restated bytes."""
import ctypes as C
import os
import tempfile
import zlib

import numpy as np
import pytest

import crop_oracle as K
import pil_bicubic_oracle as B
import pil_resize_oracle as P
import yuv_oracle as Y

pytestmark = pytest.mark.gpu

MEAN = [123.675, 116.28, 103.53, 64.0]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375, 1 / 40.0]
BICUBIC = 3
# (pixel format, channels)
LAYOUTS = {"c1": (K.INTERLEAVED, 1), "c2": (K.INTERLEAVED, 2), "c3": (K.INTERLEAVED, 3), "c4": (K.INTERLEAVED, 4),
           "nv12": (Y.NV12, 3), "i420": (Y.I420, 3)}


def _images(sizes, c, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, c), dtype=np.uint8) for h, w in sizes]


def _frame_bytes(fmt, c, h, w):
    return h * w * c if fmt == K.INTERLEAVED else h * w * 3 // 2


# ---------------------------------------------------------------------------------------------- 1. kernels
def _run_crops(frames, fmt, c, boxes, s, oh, ow, max_hw, filt=BICUBIC):
    """uint8 [len(boxes), oh, ow, c] of b200_image_crop_resize_run, with a workspace from the filter-aware query."""
    import torch
    from anakin_b200 import api, saber_abi as A
    from gpu_util import ptr, stream_ptr
    lib = A.load()
    pix, hw = api.pack_images(frames)
    offs = np.concatenate([[0], np.cumsum([_frame_bytes(fmt, c, h, w) for h, w in hw.tolist()])])
    table = (A.ImageCropEntry * len(boxes))()
    for i, (f, t, l, h, w) in enumerate(boxes):
        v = [C.c_int32() for _ in range(4)]
        A.check(lib.b200_image_resize_geometry_ex(h, w, s, oh, ow, filt, *[C.byref(x) for x in v]), "geometry")
        e = table[i]
        e.r.offset, e.r.h, e.r.w = int(offs[f]), h, w
        e.r.rh, e.r.rw, e.r.top, e.r.left = [x.value for x in v]
        e.frame_h, e.frame_w = [int(x) for x in hw[f]]
        e.box_top, e.box_left = t, l
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = len(boxes), c, oh, ow
    nbytes = C.c_size_t()
    A.check(lib.b200_image_resize_workspace(C.byref(d), filt, max_hw[0], max_hw[1], s, C.byref(nbytes)), "workspace")
    ws = torch.full((nbytes.value,), 0xA5, dtype=torch.uint8, device="cuda")
    src = torch.from_numpy(pix).cuda()
    tab = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).cuda()
    out = torch.full((len(boxes), oh, ow, c), 7, dtype=torch.uint8, device="cuda")
    A.check(lib.b200_image_crop_resize_run(C.byref(d), filt, fmt, max_hw[0], max_hw[1], s, ptr(src), ptr(tab), ptr(ws),
                                           ptr(out), stream_ptr()), "image_crop_resize")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _checker_frame(h, w, fmt, c):
    """The 0 / 255 checkerboard of pil_bicubic_oracle.case_image; in YUV, the same board in Y with neutral chroma, whose
    cvtColor is that board again."""
    board = B.case_image(h, w, 1, "checker", 0)[..., 0]
    if fmt == K.INTERLEAVED:
        return np.ascontiguousarray(np.repeat(board[..., None], c, axis=2))
    return Y.make_frame(board, np.full((h // 2, w // 2), 128, np.uint8), np.full((h // 2, w // 2), 128, np.uint8), fmt)


# frames: noise for the designed boxes (odd offsets and sizes, 1 x 1, edge-touching, the whole frame); a tall frame
# whose boxes sit on both sides of Pillow's pass-order switch; a 2 x 16384 frame whose first row, stretched to 224, has
# the longest tap records the 16384-pixel limit allows; a checkerboard whose 5x upscale overshoots in both passes; and
# the golden fixture's 375 x 500 and 3024 x 4032 photos.
FRAME_SIZES = [(300, 400), (2100, 40), (2, 16384), (46, 40), (376, 500), (3024, 4032)]
BOXES = (K.designed_boxes(300, 400)
         + [(1, 50, 7, 2000, 16), (1, 3, 11, 1600, 16), (1, 0, 0, 2100, 40), (1, 1, 1, 2001, 8)]
         + [(2, 0, 0, 1, 16384), (2, 1, 3, 1, 16380), (2, 0, 0, 2, 16384)]
         + [(3, 0, 0, 45, 40), (3, 1, 1, 44, 38)]
         + [(4, 0, 0, 375, 500), (4, 1, 0, 375, 500), (5, 0, 0, 3024, 4032)])
MAX_HW = (3024, 16384)


def _frames(layout, seed):
    fmt, c = LAYOUTS[layout]
    fr = [K.random_frame(h, w, fmt, c, seed * 10 + i) for i, (h, w) in enumerate(FRAME_SIZES)]
    fr[3] = _checker_frame(*FRAME_SIZES[3], fmt, c)
    return fr


def test_designed_boxes_cover_both_pass_orders_and_the_longest_records():
    tall = [b for b in BOXES if b[0] == 1]
    assert {P.vertical_first(h, w, 224) for _, _, _, h, w in tall} == {True, False}
    assert any(w == 16384 and h == 1 for _, _, _, h, w in BOXES)
    assert any(t % 2 and l % 2 for _, t, l, _, _ in BOXES)


@pytest.mark.parametrize("net_hw", [(224, 224), (224, 221), (200, 160)])
@pytest.mark.parametrize("s", [0, 256])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_kernel_equals_restatement(layout, s, net_hw):
    """Every box of every frame in one launch (221: the byte-store instance of the second pass)."""
    fmt, c = LAYOUTS[layout]
    oh, ow = net_hw
    frames = _frames(layout, zlib.crc32(repr((layout, s)).encode()) % 1000)
    got = _run_crops(frames, fmt, c, BOXES, s, oh, ow, MAX_HW)
    for i, box in enumerate(BOXES):
        want = B.resize_u8(K.crop(frames, fmt, box), s, oh, ow)
        assert np.array_equal(got[i], want), (layout, box, int(np.abs(got[i].astype(int) - want).max()))


def test_kernel_pass_orders_and_overshoot_are_pillows():
    """The restatement run the other way differs on the tall boxes and the clamp is active on the checkerboard, so the
    kernel's agreement above pins both rules."""
    fmt, c = LAYOUTS["c3"]
    frames = _frames("c3", 3)
    boxes = [(1, 50, 7, 2000, 16), (1, 3, 11, 1600, 16), (3, 0, 0, 45, 40)]
    got = _run_crops(frames, fmt, c, boxes, 0, 224, 200, MAX_HW)
    for i, box in enumerate(boxes[:2]):
        img = K.crop(frames, fmt, box)
        vf = P.vertical_first(box[3], box[4], 224)
        assert np.array_equal(got[i], B.resize_u8(img, 0, 224, 200))
        assert not np.array_equal(got[i], B.resize_u8(img, 0, 224, 200, vfirst=not vf))
    sums = []
    want = B.resize_u8(K.crop(frames, fmt, boxes[2]), 0, 224, 200, sums=sums)
    assert all(a.min() < 0 and a.max() > 255 << B.PRECISION_BITS for a in sums)
    assert np.array_equal(got[2], want)


def test_kernel_filters_do_not_share_state():
    """The same frames and workspace sizes through filters 1 and 3 alternately: each gives its own restatement."""
    fmt, c = LAYOUTS["nv12"]
    frames = _frames("nv12", 5)
    boxes = K.designed_boxes(300, 400) + [(4, 0, 0, 375, 500)]
    for filt, oracle in ((BICUBIC, B), (1, P), (BICUBIC, B)):
        got = _run_crops(frames, fmt, c, boxes, 256, 224, 224, MAX_HW, filt=filt)
        for i, box in enumerate(boxes):
            assert np.array_equal(got[i], oracle.resize_u8(K.crop(frames, fmt, box), 256, 224, 224)), (filt, box)


# ---------------------------------------------------------------------------------------------- 2. Net
def _graphs(g_dict, batch, max_hw, resize_short, filt="pil_bicubic"):
    """(plain image Graph, resizing image Graph with `filt`) from one model dict."""
    from anakin_b200 import anakin_bin, api
    blob = anakin_bin.dumps(g_dict)
    Gp, Gr = api.Graph.from_bytes(blob), api.Graph.from_bytes(blob)
    for G in (Gp, Gr):
        G.set_input_image("input_0", MEAN[:3], SCALE[:3], [2, 1, 0])
    Gr.set_input_image_resize("input_0", max_hw[0], max_hw[1], resize_short, filter=filt)
    for G in (Gp, Gr):
        G.ResetBatchSize("input_0", batch)
        G.Optimize()
    return Gp, Gr


def compare_nets(model, precision, batch, resize_short, size_sets, max_hw):
    """A Net with the bicubic filter, one with the bilinear filter and the plain image Net: the resizing Nets' input
    tensors hold their own filter's restated bytes, and each gives the plain Net's outputs for those bytes."""
    from anakin_b200 import api, modelzoo, saber_abi
    g_dict = modelzoo.build(model, batch=batch, precision=precision)
    shape = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"]
    H, W = shape[2], shape[3]
    Gp, Gb = _graphs(g_dict, batch, max_hw, resize_short)
    _, Gl = _graphs(g_dict, batch, max_hw, resize_short, filt="pil")
    np_, nb, nl = api.Net(Gp, precision), api.Net(Gb, precision), api.Net(Gl, precision)
    assert nb.exec_order()[0] == ["input_0", "ImageResize"] and nb.exec_order()[1:] == np_.exec_order()
    lib = saber_abi.load()
    for it, sizes in enumerate(size_sets):
        imgs = _images(sizes, 3, seed=1000 * it + batch)
        for net, oracle, name in ((nb, B, "bicubic"), (nl, P, "bilinear")):
            want_in = oracle.resize_batch(imgs, resize_short, H, W)
            np_.set_input_image("input_0", want_in)
            net.set_input_images("input_0", imgs)
            n0 = lib.b200_launch_count()
            net.prediction()
            n1 = lib.b200_launch_count()
            np_.prediction()
            n2 = lib.b200_launch_count()
            np_.sync(); net.sync()
            if it == 0:     # eager: taps, first pass, second pass
                assert n1 - n0 == n2 - n1 + 3, (name, n1 - n0, n2 - n1)
            assert np.array_equal(net.read_tensor("input_0")[0], want_in), (model, precision, name, it)
            for out in np_.out_names:
                a, b = np_.get_output(out), net.get_output(out)
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (model, precision, name, out, it)
    assert nb.cuda_graph_active() and nl.cuda_graph_active()


TINY_SETS = [[(32, 32), (75, 41)], [(1, 1), (80, 96)], [(33, 64), (96, 17)], [(96, 96), (5, 90)]]


@pytest.mark.parametrize("precision", ["fp32", "int8"])
def test_tiny_resnet_bicubic_bit_exact(precision):
    compare_nets("tiny_resnet", precision, 2, 36, TINY_SETS, (96, 96))


BIG = [(375, 500), (500, 375), (480, 640), (960, 1280), (224, 224), (100, 150), (333, 517), (3024, 4032)]


def test_resnet50_int8_bicubic_bit_exact():
    compare_nets("resnet50", "int8", 8, 256, [BIG, BIG[::-1]], (3024, 4032))


def test_net_workspace_is_the_bicubic_query():
    """The Net sizes its workspace through b200_image_resize_workspace: a graph at the 16384-pixel limit builds, and
    its widest request (a 1 x 16384 image, 292 taps per column) is resized bit for bit."""
    from anakin_b200 import api, modelzoo
    Gp, Gb = _graphs(modelzoo.build("tiny_resnet", 2, precision="int8"), 2, (16384, 16384), 0)
    nb, np_ = api.Net(Gb, "int8"), api.Net(Gp, "int8")
    imgs = _images([(1, 16384), (16384, 3)], 3, seed=4)
    nb.set_input_images("input_0", imgs)
    nb.prediction(); nb.sync()
    want_in = B.resize_batch(imgs, 0, 32, 32)
    assert np.array_equal(nb.read_tensor("input_0")[0], want_in)
    np_.set_input_image("input_0", want_in)
    np_.prediction(); np_.sync()
    assert np.array_equal(np_.get_output(np_.out_names[0]), nb.get_output(nb.out_names[0]))


def test_net_crops_of_yuv_frames():
    """An NV12 crops Net with the bicubic filter: each box, odd offsets included, is the restatement of the box cut
    from the frame's cvtColor."""
    from anakin_b200 import api, modelzoo
    g = modelzoo.build("tiny_resnet", 4, precision="int8")
    from anakin_b200 import anakin_bin
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.set_input_image("input_0", MEAN[:3], SCALE[:3], [2, 1, 0])
    G.set_input_image_resize("input_0", 96, 96, 36, filter="pil_bicubic", pixel_format="nv12")
    G.ResetBatchSize("input_0", 4)
    G.Optimize()
    net = api.Net(G, "int8")
    f = [Y.random_frame(h, w, Y.NV12, 60 + i) for i, (h, w) in enumerate([(96, 96), (40, 76)])]
    reqs = [[(0, 1, 3, 5, 7), (0, 0, 0, 96, 96), (1, 3, 3, 37, 73), (1, 0, 1, 1, 1)],
            [(1, 0, 0, 40, 76), (0, 17, 9, 61, 33), (0, 95, 95, 1, 1), (1, 1, 5, 2, 70)]]
    for boxes in reqs:
        net.set_input_crops("input_0", f, boxes)
        net.prediction(); net.sync()
        want = np.stack([B.resize_u8(K.crop(f, Y.NV12, b), 36, 32, 32) for b in boxes])
        assert np.array_equal(net.read_tensor("input_0")[0], want), boxes


# ---------------------------------------------------------------------------------------------- 3. Worker
def test_batching_worker_bicubic_rows_equal_a_plain_net():
    """A batching Worker (max_delay_us) serving bicubic requests of k < batch images: each request's rows equal those
    of the plain image Net fed the restated bytes."""
    import threading
    import torch
    from anakin_b200 import anakin_bin, api, modelzoo
    batch = 4
    g = modelzoo.build("tiny_resnet", batch=batch, precision="int8")
    blob = anakin_bin.dumps(g)
    G, Gp = api.Graph.from_bytes(blob), api.Graph.from_bytes(blob)
    for X in (G, Gp):
        X.set_input_image("input_0", MEAN[:3], SCALE[:3], [2, 1, 0])
    G.set_input_image_resize("input_0", 96, 96, 36, filter="pil_bicubic")
    for X in (G, Gp):
        X.ResetBatchSize("input_0", batch)
    rng = np.random.default_rng(21)
    src = [(32, 32), (75, 41), (1, 1), (80, 96), (33, 64), (96, 17), (96, 96), (50, 50), (17, 90), (41, 39)]
    reqs = []
    for i, k in enumerate(int(k) for k in rng.integers(1, batch, 24)):       # k < batch
        imgs = _images([src[j] for j in rng.integers(0, len(src), k)], 3, seed=200 + i)
        pix, hw = api.pack_images(imgs)
        reqs.append((k, imgs, torch.from_numpy(pix).pin_memory(), torch.from_numpy(hw).pin_memory()))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "bicubic.anakin.bin")
        G.save(path)
        Gp.Optimize()
        plain = api.Net(Gp, "int8")
        w = api.Worker(path, "int8", threads=2, devices=(0,), max_delay_us=200)
        out_floats = w.image_sizes()["output"]
        outs = [torch.zeros(out_floats * k, dtype=torch.float32).pin_memory() for k, *_ in reqs]
        errors = []

        def client(ids):
            try:
                for i in ids:
                    _, _, pix, hw = reqs[i]
                    w.async_prediction_images_ptr(pix.data_ptr(), pix.numel(), hw.data_ptr(), hw.shape[0],
                                                  outs[i].data_ptr(), outs[i].numel())
                for _ in ids:
                    w.async_get_result()
            except Exception as e:      # reported by the main thread
                errors.append(e)

        threads = [threading.Thread(target=client, args=(list(range(c, len(reqs), 3)),)) for c in range(3)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        del w
    assert not errors, errors
    filler = B.resize_batch(_images([(20, 20)] * batch, 3, seed=9), 36, 32, 32)
    for i, (k, imgs, _, _) in enumerate(reqs):
        x = filler.copy()
        x[:k] = B.resize_batch(imgs, 36, 32, 32)
        plain.set_input_image("input_0", x)
        plain.prediction(); plain.sync()
        want = plain.read_tensor(plain.out_names[0])[0].reshape(batch, -1)[:k]
        got = outs[i].numpy()
        assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(want, np.float32).reshape(-1).view(np.uint32)), i
