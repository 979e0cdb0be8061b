"""GPU: OpenCV's INTER_LINEAR filter of the on-device resize (b200_image_crop_resize_run with
B200_IMAGE_RESIZE_CV2_LINEAR, the `<input>:ImageResize` op with image_resize_filter 5). Every comparison is bit for bit,
with deterministic seeds: the kernel against the numpy restatement (tests/cv2_resize_oracle.py, pinned to cv2 by
tests/test_cpu_image_resize_cv2.py) applied to each box cut out of its frame (the cvtColor image for NV12 / I420);
Nets and a batching Worker with the filter against the plain image Net fed the restated bytes."""
import ctypes as C
import os
import tempfile
import zlib

import numpy as np
import pytest

import crop_oracle as K
import cv2_resize_oracle as O
import yuv_oracle as Y

pytestmark = pytest.mark.gpu

MEAN = [123.675, 116.28, 103.53]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375]
CV2_LINEAR = 5
# (pixel format, channels)
LAYOUTS = {"c1": (K.INTERLEAVED, 1), "c2": (K.INTERLEAVED, 2), "c3": (K.INTERLEAVED, 3), "c4": (K.INTERLEAVED, 4),
           "nv12": (Y.NV12, 3), "i420": (Y.I420, 3)}


def _images(sizes, c, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, c), dtype=np.uint8) for h, w in sizes]


def _frame_bytes(fmt, c, h, w):
    return h * w * c if fmt == K.INTERLEAVED else h * w * 3 // 2


# ---------------------------------------------------------------------------------------------- 1. kernel
def _run_crops(frames, fmt, c, boxes, s, oh, ow, filt=CV2_LINEAR):
    """uint8 [len(boxes), oh, ow, c] of b200_image_crop_resize_run; the filter takes no workspace."""
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
    src = torch.from_numpy(pix).cuda()
    tab = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).cuda()
    out = torch.full((len(boxes), oh, ow, c), 7, dtype=torch.uint8, device="cuda")
    A.check(lib.b200_image_crop_resize_run(C.byref(d), filt, fmt, 0, 0, s, ptr(src), ptr(tab), None, ptr(out),
                                           stream_ptr()), "image_crop_resize")
    torch.cuda.synchronize()
    return out.cpu().numpy()


# frames: noise for the designed boxes (odd offsets and sizes, 1 x 1, edge-touching, the whole frame: most of them
# upscale); a 448 x 448 frame whose whole box and 448 x 442 box shrink exactly 2x to 224 x 224 and 224 x 221; a
# 2 x 16384 strip; the 375 x 500 and 3024 x 4032 photos
FRAME_SIZES = [(300, 400), (448, 448), (2, 16384), (376, 500), (3024, 4032)]
BOXES = (K.designed_boxes(300, 400)
         + [(1, 0, 0, 448, 448), (1, 0, 6, 448, 442), (1, 1, 1, 446, 445)]
         + [(2, 0, 0, 1, 16384), (2, 1, 3, 1, 16380), (2, 0, 0, 2, 16384)]
         + [(3, 0, 0, 375, 500), (3, 1, 0, 375, 500), (4, 0, 0, 3024, 4032)])


def _frames(layout, seed):
    fmt, c = LAYOUTS[layout]
    return [K.random_frame(h, w, fmt, c, seed * 10 + i) for i, (h, w) in enumerate(FRAME_SIZES)]


def _restated(frames, fmt, boxes, s, oh, ow):
    """The restatement of every box, each frame converted to RGB once."""
    rgb = [K.frame_rgb(f, fmt) for f in frames]
    return [O.resize_u8(rgb[f][t:t + h, l:l + w], s, oh, ow) for f, t, l, h, w in boxes]


@pytest.mark.parametrize("net_hw", [(224, 224), (224, 221), (200, 160)])
@pytest.mark.parametrize("s", [0, 256])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_kernel_equals_restatement(layout, s, net_hw):
    """Every box of every frame in one launch (221: the byte-store instance)."""
    fmt, c = LAYOUTS[layout]
    oh, ow = net_hw
    frames = _frames(layout, zlib.crc32(repr((layout, s)).encode()) % 1000)
    got = _run_crops(frames, fmt, c, BOXES, s, oh, ow)
    for i, (box, want) in enumerate(zip(BOXES, _restated(frames, fmt, BOXES, s, oh, ow))):
        assert np.array_equal(got[i], want), (layout, box, int(np.abs(got[i].astype(int) - want).max()))


def test_kernel_two_channel_2x_shrink_rounds_half_to_even():
    """Exact 2x shrinks with c = 2 take the half-to-even mean and every other c the (sum + 2) >> 2 one; the designed
    frame has block sums at every residue mod 4, so the two rules differ on it and the kernel must pick each."""
    rng = np.random.default_rng(3)
    for c in (1, 2, 3, 4):
        frame = rng.integers(0, 256, (448, 448, c), dtype=np.uint8)
        got = _run_crops([frame], K.INTERLEAVED, c, [(0, 0, 0, 448, 448)], 0, 224, 224)[0]
        v = frame.astype(np.int64).reshape(224, 2, 224, 2, c).sum(axis=(1, 3))
        assert {int(r) for r in np.unique(v & 3)} == {0, 1, 2, 3}
        half_even, half_up = (v + 1 + ((v >> 2) & 1)) >> 2, (v + 2) >> 2
        assert np.array_equal(got, half_even if c == 2 else half_up), c
        assert not np.array_equal(half_even, half_up)


def test_kernel_filters_do_not_share_state():
    """The same frames through the reference filter and cv2's alternately: each gives its own bytes."""
    import image_resize_oracle as R
    fmt, c = LAYOUTS["i420"]
    frames = _frames("i420", 5)
    boxes = K.designed_boxes(300, 400) + [(3, 0, 0, 375, 500)]
    rgb = [K.frame_rgb(f, fmt) for f in frames]
    for filt in (CV2_LINEAR, 0, CV2_LINEAR):
        got = _run_crops(frames, fmt, c, boxes, 256, 224, 224, filt=filt)
        for i, (f, t, l, h, w) in enumerate(boxes):
            img = rgb[f][t:t + h, l:l + w]
            want = O.resize_u8(img, 256, 224, 224) if filt == CV2_LINEAR else R.image_resize_u8(img, 256, 224, 224)
            assert np.array_equal(got[i], want), (filt, boxes[i])


# ---------------------------------------------------------------------------------------------- 2. Net
def _graphs(g_dict, batch, max_hw, resize_short, pixel_format="interleaved", optimize=True):
    """(plain image Graph, resizing image Graph with the cv2 filter) from one model dict."""
    from anakin_b200 import anakin_bin, api
    blob = anakin_bin.dumps(g_dict)
    Gp, Gr = api.Graph.from_bytes(blob), api.Graph.from_bytes(blob)
    for G in (Gp, Gr):
        G.set_input_image("input_0", MEAN, SCALE, [2, 1, 0])
    Gr.set_input_image_resize("input_0", max_hw[0], max_hw[1], resize_short, filter="cv2_linear",
                              pixel_format=pixel_format)
    for G in (Gp, Gr):
        G.ResetBatchSize("input_0", batch)
        if optimize:
            G.Optimize()
    return Gp, Gr


def compare_nets(model, precision, batch, resize_short, size_sets, max_hw):
    """The cv2-filter Net's input tensor holds the restated bytes, and it gives the plain Net's outputs for them, with
    one launch for the resize."""
    from anakin_b200 import api, modelzoo, saber_abi
    g_dict = modelzoo.build(model, batch=batch, precision=precision)
    shape = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"]
    H, W = shape[2], shape[3]
    Gp, Gr = _graphs(g_dict, batch, max_hw, resize_short)
    np_, nr = api.Net(Gp, precision), api.Net(Gr, precision)
    assert nr.exec_order()[0] == ["input_0", "ImageResize"] and nr.exec_order()[1:] == np_.exec_order()
    lib = saber_abi.load()
    for it, sizes in enumerate(size_sets):
        imgs = _images(sizes, 3, seed=1000 * it + batch)
        want_in = O.resize_batch(imgs, resize_short, H, W)
        np_.set_input_image("input_0", want_in)
        nr.set_input_images("input_0", imgs)
        n0 = lib.b200_launch_count()
        nr.prediction()
        n1 = lib.b200_launch_count()
        np_.prediction()
        n2 = lib.b200_launch_count()
        np_.sync(); nr.sync()
        if it == 0:     # eager: one resize launch
            assert n1 - n0 == n2 - n1 + 1, (n1 - n0, n2 - n1)
        assert np.array_equal(nr.read_tensor("input_0")[0], want_in), (model, precision, it)
        for out in np_.out_names:
            a, b = np_.get_output(out), nr.get_output(out)
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (model, precision, out, it)
    assert nr.cuda_graph_active()


TINY_SETS = [[(32, 32), (75, 41)], [(1, 1), (80, 96)], [(64, 72), (96, 17)], [(96, 96), (5, 90)]]


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_tiny_resnet_cv2_bit_exact(precision):
    compare_nets("tiny_resnet", precision, 2, 36, TINY_SETS, (96, 96))


BIG = [(375, 500), (500, 375), (480, 640), (960, 1280), (224, 224), (512, 600), (333, 517), (3024, 4032)]


def test_resnet50_int8_cv2_bit_exact():
    compare_nets("resnet50", "int8", 8, 256, [BIG, BIG[::-1]], (3024, 4032))


def test_net_crops_of_nv12_frames():
    """An NV12 crops Net with the cv2 filter: each box, odd offsets and upscales included, is the restatement of the box
    cut from the frame's cvtColor."""
    from anakin_b200 import api, modelzoo
    _, G = _graphs(modelzoo.build("tiny_resnet", 4, precision="int8"), 4, (96, 96), 36, pixel_format="nv12")
    net = api.Net(G, "int8")
    f = [Y.random_frame(h, w, Y.NV12, 60 + i) for i, (h, w) in enumerate([(96, 96), (40, 76)])]
    reqs = [[(0, 1, 3, 5, 7), (0, 0, 0, 96, 96), (1, 3, 3, 37, 73), (1, 0, 1, 1, 1)],
            [(1, 0, 0, 40, 76), (0, 17, 9, 61, 33), (0, 95, 95, 1, 1), (1, 1, 5, 2, 70)]]
    for boxes in reqs:
        net.set_input_crops("input_0", f, boxes)
        net.prediction(); net.sync()
        assert np.array_equal(net.read_tensor("input_0")[0], np.stack(_restated(f, Y.NV12, boxes, 36, 32, 32))), boxes


# ---------------------------------------------------------------------------------------------- 3. Worker
def test_batching_worker_cv2_rows_equal_a_plain_net():
    """A batching Worker (max_delay_us) serving cv2-filter requests of k < batch images: each request's rows equal
    those of the plain image Net fed the restated bytes."""
    import threading
    import torch
    from anakin_b200 import api, modelzoo
    batch = 4
    Gp, G = _graphs(modelzoo.build("tiny_resnet", batch=batch, precision="int8"), batch, (96, 96), 36, optimize=False)
    rng = np.random.default_rng(22)
    src = [(32, 32), (75, 41), (1, 1), (80, 96), (64, 72), (96, 17), (96, 96), (50, 50), (17, 90), (41, 39)]
    reqs = []
    for i, k in enumerate(int(k) for k in rng.integers(1, batch, 24)):       # k < batch
        imgs = _images([src[j] for j in rng.integers(0, len(src), k)], 3, seed=300 + i)
        pix, hw = api.pack_images(imgs)
        reqs.append((k, imgs, torch.from_numpy(pix).pin_memory(), torch.from_numpy(hw).pin_memory()))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "cv2.anakin.bin")
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
    filler = O.resize_batch(_images([(20, 20)] * batch, 3, seed=9), 36, 32, 32)
    for i, (k, imgs, _, _) in enumerate(reqs):
        x = filler.copy()
        x[:k] = O.resize_batch(imgs, 36, 32, 32)
        plain.set_input_image("input_0", x)
        plain.prediction(); plain.sync()
        want = plain.read_tensor(plain.out_names[0])[0].reshape(batch, -1)[:k]
        got = outs[i].numpy()
        assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(want, np.float32).reshape(-1).view(np.uint32)), i
