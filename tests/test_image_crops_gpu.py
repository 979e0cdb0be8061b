"""GPU: boxes cropped out of frames by the on-device resize (b200_image_crop_resize_run, Net.set_input_crops, the
Worker's crops requests). Every comparison is bit for bit, with deterministic seeds: the kernel against the crop
restatement (tests/crop_oracle.py, pinned to Pillow, torchvision and OpenCV by tests/test_cpu_image_crops.py), against
itself on frames altered outside every box, and against the whole-image entry points; a crops Net against the
interleaved resize Net fed the crops cut on the host."""
import ctypes as C
import os
import tempfile
import zlib

import numpy as np
import pytest

import crop_oracle as K
import yuv_oracle as Y

pytestmark = pytest.mark.gpu

MEAN = [123.675, 116.28, 103.53, 64.0]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375, 1 / 40.0]
FILTERS = {"reference": 0, "pil": 1}
# (pixel format, channels)
LAYOUTS = {"c1": (K.INTERLEAVED, 1), "c3": (K.INTERLEAVED, 3), "c4": (K.INTERLEAVED, 4), "nv12": (Y.NV12, 3),
           "i420": (Y.I420, 3)}


def _frame_bytes(fmt, c, h, w):
    return h * w * c if fmt == K.INTERLEAVED else h * w * 3 // 2


# ---------------------------------------------------------------------------------------------- kernels
def _run_crops(frames, fmt, c, boxes, filt, s, oh, ow, max_hw):
    """uint8 [len(boxes), oh, ow, c] of b200_image_crop_resize_run."""
    import torch
    from anakin_b200 import api, saber_abi as A
    from gpu_util import ptr, stream_ptr
    lib = A.load()
    pix, hw = api.pack_images(frames)
    offs = np.concatenate([[0], np.cumsum([_frame_bytes(fmt, c, h, w) for h, w in hw.tolist()])])
    table = (A.ImageCropEntry * len(boxes))()
    for i, (f, t, l, h, w) in enumerate(boxes):
        v = [C.c_int32() for _ in range(4)]
        A.check(lib.b200_image_resize_geometry_ex(h, w, s, oh, ow, FILTERS[filt], *[C.byref(x) for x in v]), "geometry")
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
    ws = None
    if filt == "pil":
        nbytes = C.c_size_t()
        A.check(lib.b200_image_resize_pil_workspace(C.byref(d), max_hw[0], max_hw[1], s, C.byref(nbytes)), "workspace")
        ws = torch.full((nbytes.value,), 0xA5, dtype=torch.uint8, device="cuda")
    A.check(lib.b200_image_crop_resize_run(C.byref(d), FILTERS[filt], fmt, max_hw[0], max_hw[1], s, ptr(src), ptr(tab),
                                           ptr(ws), ptr(out), stream_ptr()), "image_crop_resize")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _run_whole(frames, fmt, c, filt, s, oh, ow, max_hw):
    """The same frames through the whole-image entry points of their filter and layout."""
    import torch
    from anakin_b200 import api, saber_abi as A
    from gpu_util import ptr, stream_ptr
    lib = A.load()
    pix, hw = api.pack_images(frames)
    table = (A.ImageResizeEntry * len(frames))()
    off = 0
    for i, (h, w) in enumerate(hw.tolist()):
        v = [C.c_int32() for _ in range(4)]
        A.check(lib.b200_image_resize_geometry_ex(h, w, s, oh, ow, FILTERS[filt], *[C.byref(x) for x in v]), "geometry")
        table[i].offset, table[i].h, table[i].w = off, h, w
        table[i].rh, table[i].rw, table[i].top, table[i].left = [x.value for x in v]
        off += _frame_bytes(fmt, c, h, w)
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = len(frames), c, oh, ow
    src = torch.from_numpy(pix).cuda()
    tab = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).cuda()
    out = torch.full((len(frames), oh, ow, c), 7, dtype=torch.uint8, device="cuda")
    st = stream_ptr()
    if filt == "pil":
        nbytes = C.c_size_t()
        A.check(lib.b200_image_resize_pil_workspace(C.byref(d), max_hw[0], max_hw[1], s, C.byref(nbytes)), "workspace")
        ws = torch.full((nbytes.value,), 0xA5, dtype=torch.uint8, device="cuda")
        if fmt == K.INTERLEAVED:
            rc = lib.b200_image_resize_pil_run(C.byref(d), max_hw[0], max_hw[1], s, ptr(src), ptr(tab), ptr(ws),
                                               ptr(out), st)
        else:
            rc = lib.b200_image_resize_pil_yuv_run(C.byref(d), fmt, max_hw[0], max_hw[1], s, ptr(src), ptr(tab),
                                                   ptr(ws), ptr(out), st)
    elif fmt == K.INTERLEAVED:
        rc = lib.b200_image_resize_run(C.byref(d), ptr(src), ptr(tab), ptr(out), st)
    else:
        rc = lib.b200_image_resize_yuv_run(C.byref(d), fmt, ptr(src), ptr(tab), ptr(out), st)
    A.check(rc, "image_resize")
    torch.cuda.synchronize()
    return out.cpu().numpy()


# frames 0..2, and boxes of all of them in one launch: the designed boxes of frame 0, a few of frame 1, and tall thin
# boxes on both sides of Pillow's pass-order switch in frame 2 (the frame itself is on neither side)
FRAME_SIZES = [(300, 400), (120, 90), (2100, 40)]
BOXES = (K.designed_boxes(300, 400) + K.designed_boxes(120, 90, f=1)[2:6]
         + [(2, 50, 7, 2000, 16), (2, 3, 11, 1600, 16), (2, 0, 0, 2100, 40), (0, 17, 33, 250, 111)])
MAX_HW = (2100, 400)


def _frames(layout, seed):
    fmt, c = LAYOUTS[layout]
    return [K.random_frame(h, w, fmt, c, seed * 10 + i) for i, (h, w) in enumerate(FRAME_SIZES)]


@pytest.mark.parametrize("net_hw", [(224, 224), (200, 160)])
@pytest.mark.parametrize("s", [0, 232, 256])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("filt", ["reference", "pil"])
def test_kernel_equals_restatement(filt, layout, s, net_hw):
    fmt, c = LAYOUTS[layout]
    oh, ow = net_hw
    frames = _frames(layout, zlib.crc32(repr((filt, layout, s, net_hw)).encode()))
    for w_out in [ow] + ([222] if net_hw == (224, 224) else []):     # 222: the byte-store instance
        got = _run_crops(frames, fmt, c, BOXES, filt, s, oh, w_out, MAX_HW)
        for i, box in enumerate(BOXES):
            want = K.resize_box(frames, fmt, box, filt, s, oh, w_out)
            assert np.array_equal(got[i], want), (box, w_out, int(np.abs(got[i].astype(int) - want).max()))


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("filt", ["reference", "pil"])
def test_no_tap_outside_the_box(filt, layout):
    """Every byte no box may read is replaced (tests/crop_oracle.py outside_altered): the results stay the same. Each
    frame keeps only its own boxes, so the boxes that touch a frame edge are the only protection of that edge."""
    fmt, c = LAYOUTS[layout]
    frames = _frames(layout, 77)
    for boxes in ([b for b in BOXES if b[3] * b[4] < 20000], [(0, 1, 3, 151, 201), (1, 7, 5, 33, 19), (2, 9, 1, 2000, 37)]):
        altered = [K.outside_altered(f, fmt, [b for b in boxes if b[0] == i]) for i, f in enumerate(frames)]
        for s in (0, 256):
            a = _run_crops(frames, fmt, c, boxes, filt, s, 224, 224, MAX_HW)
            b = _run_crops(altered, fmt, c, boxes, filt, s, 224, 224, MAX_HW)
            assert np.array_equal(a, b), (s, [i for i in range(len(boxes)) if not np.array_equal(a[i], b[i])])


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("filt", ["reference", "pil"])
def test_whole_frame_boxes_equal_the_image_entry_points(filt, layout):
    fmt, c = LAYOUTS[layout]
    frames = _frames(layout, 5) + [K.random_frame(2, 2, fmt, c, 3), K.random_frame(1080, 1920, fmt, c, 4)]
    boxes = [(i,) + (0, 0) + K.frame_hw(f, fmt) for i, f in enumerate(frames)]
    max_hw = (2100, 1920)
    for s, (oh, ow) in ((256, (224, 224)), (0, (200, 160)), (232, (224, 222))):
        assert np.array_equal(_run_crops(frames, fmt, c, boxes, filt, s, oh, ow, max_hw),
                              _run_whole(frames, fmt, c, filt, s, oh, ow, max_hw)), s


# ---------------------------------------------------------------------------------------------- Net
def _graph(g_dict, batch, max_hw, resize_short, filt, pixel_format, c=3):
    from anakin_b200 import anakin_bin, api
    G = api.Graph.from_bytes(anakin_bin.dumps(g_dict))
    G.set_input_image("input_0", MEAN[:c], SCALE[:c], list(range(c)))
    G.set_input_image_resize("input_0", max_hw[0], max_hw[1], resize_short, filter=filt, pixel_format=pixel_format)
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    return G


def compare_nets(model, precision, batch, resize_short, requests, max_hw, filt, name, exports=None, check_graph=False):
    """A crops Net of layout `name` and the interleaved resize Net fed the crops cut on the host: the same outputs,
    exports and input tensor bit for bit, and the same launches, for every request: (frames, boxes), or (frames, None)
    for an images request."""
    from anakin_b200 import api, modelzoo, saber_abi
    fmt = K.FORMATS[name]
    g_dict = modelzoo.build(model, batch=batch, precision=precision)
    shape = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"]
    H, W = shape[2], shape[3]
    nc = api.Net(_graph(g_dict, batch, max_hw, resize_short, filt, name), precision, exports=exports)
    ni = api.Net(_graph(g_dict, batch, max_hw, resize_short, filt, "interleaved"), precision, exports=exports)
    lib = saber_abi.load()
    for it, (frames, boxes) in enumerate(requests):
        if boxes is None:
            nc.set_input_images("input_0", frames)
            boxes = [(i, 0, 0) + K.frame_hw(f, fmt) for i, f in enumerate(frames)]
        else:
            nc.set_input_crops("input_0", frames, boxes)
        ni.set_input_images("input_0", [K.crop(frames, fmt, b) for b in boxes])
        n0 = lib.b200_launch_count()
        nc.prediction()
        n1 = lib.b200_launch_count()
        ni.prediction()
        n2 = lib.b200_launch_count()
        ni.sync(); nc.sync()
        assert n1 - n0 == n2 - n1, (n1 - n0, n2 - n1)
        if check_graph and it >= 2:
            assert nc.cuda_graph_active() and n1 == n0, (it, n1 - n0)
        want_in = K.resize_boxes(frames, fmt, boxes, filt, resize_short, H, W)
        assert np.array_equal(nc.read_tensor("input_0")[0], want_in), (model, precision, it)
        for nm in ni.out_names:
            assert np.array_equal(ni.get_output(nm).view(np.uint8), nc.get_output(nm).view(np.uint8)), (nm, it)
        for x in exports or []:
            assert np.array_equal(ni.get_export(x).view(np.uint32), nc.get_export(x).view(np.uint32)), (x, it)
    assert nc.cuda_graph_active()


def _tiny_requests(fmt, seed):
    frames = [K.random_frame(h, w, fmt, 3, seed + i) for i, (h, w) in enumerate([(96, 80), (40, 64), (2, 2)])]
    return [([frames[0]], [(0, 1, 3, 61, 29), (0, 0, 0, 96, 80)]),
            (frames[:2], [(1, 5, 7, 1, 1), (0, 10, 11, 85, 69)]),
            ([frames[1], frames[2]], [(0, 39, 0, 1, 64), (1, 0, 1, 2, 1)])]


@pytest.mark.parametrize("precision", ["fp32", "fp16", "int8"])
@pytest.mark.parametrize("model", ["tiny_resnet", "tiny_mobilenet"])
def test_tiny_nets_equal_the_interleaved_net(model, precision):
    for filt, name in (("reference", "nv12"), ("pil", "interleaved"), ("pil", "i420")):
        compare_nets(model, precision, 2, 36, _tiny_requests(K.FORMATS[name], 3), (96, 96), filt, name)


def test_resnet50_int8_eight_boxes_of_a_1080p_nv12_frame():
    frame = Y.random_frame(1080, 1920, Y.NV12, 11)
    boxes = [(0, 0, 0, 1080, 1920), (0, 101, 203, 333, 217), (0, 517, 1401, 563, 519), (0, 1, 1, 31, 47),
             (0, 700, 3, 380, 1911), (0, 0, 1919, 1080, 1), (0, 255, 640, 256, 257), (0, 1079, 0, 1, 1920)]
    compare_nets("resnet50", "int8", 8, 256, [([frame], boxes), ([frame], boxes[::-1])], (1080, 1920), "pil", "nv12",
                 exports=["pool5"])


@pytest.mark.parametrize("filt", ["reference", "pil"])
def test_one_cuda_graph_serves_images_and_crops_requests(filt):
    fmt = Y.I420
    f = [Y.random_frame(h, w, fmt, 40 + i) for i, (h, w) in enumerate([(600, 600), (32, 76), (2, 2), (590, 6)])]
    requests = [([f[0], f[1]], None), ([f[0]], [(0, 3, 5, 7, 9), (0, 0, 0, 600, 600)]),
                ([f[1], f[3]], [(1, 11, 1, 579, 5), (0, 1, 0, 31, 76)]), ([f[1], f[2]], None),
                ([f[3], f[2]], [(1, 1, 1, 1, 1), (0, 0, 0, 590, 6)]), ([f[0]], [(0, 599, 0, 1, 600), (0, 0, 599, 600, 1)])]
    compare_nets("tiny_resnet", "int8", 2, 36, requests, (600, 600), filt, "i420", check_graph=True)


def test_net_refusals():
    from anakin_b200 import api, modelzoo
    G = _graph(modelzoo.build("tiny_resnet", batch=2, precision="int8"), 2, (96, 96), 36, "reference", "nv12")
    net = api.Net(G, "int8")
    fr = [Y.random_frame(96, 80, Y.NV12, 1), Y.random_frame(40, 64, Y.NV12, 2)]
    cases = [([fr[0]], [(0, 0, 0, 96, 80)], "1 boxes, the batch is 2"),
             (fr, [(0, 0, 0, 96, 80), (2, 0, 0, 1, 1)], r"box 1 \(frame 2, top 0, left 0, 1 x 1\): no frame 2 among the "
                                                        r"request's 2"),
             (fr, [(0, 0, 0, 96, 80), (1, 1, 0, 40, 64)], r"box 1 \(frame 1, top 1, left 0, 40 x 64\) is not inside "
                                                          r"frame 1 \(40 x 64\)"),
             (fr, [(0, -1, 0, 2, 2), (1, 0, 0, 1, 1)], "box 0 .* is not inside frame 0"),
             (fr, [(0, 0, 0, 0, 2), (1, 0, 0, 1, 1)], "box 0 .* is not inside frame 0"),
             (fr + fr[:1], [(0, 0, 0, 1, 1), (1, 0, 0, 1, 1)], "3 frames for 2 boxes"),
             ([np.zeros((98 * 3 // 2, 80), np.uint8)], [(0, 0, 0, 1, 1)] * 2, "frame 0 is 98 x 80, outside 1..max")]
    for frames, boxes, msg in cases:
        with pytest.raises(api.AnakinError, match=msg):
            net.set_input_crops("input_0", frames, boxes)
    # an odd-sized frame cannot be packed from cv2's layout: the sizes table says 39 rows
    pix, _ = api.pack_images([fr[1]])
    lib = api.load()
    hw = np.array([[39, 64]], np.int32)
    bx = np.array([[0, 0, 0, 1, 1]] * 2, np.int32)
    assert lib.anakin_net_set_input_crops(net._h, b"input_0", pix.ctypes.data_as(C.c_void_p), pix.nbytes,
                                          hw.ctypes.data_as(C.c_void_p), 1, bx.ctypes.data_as(C.c_void_p), 2) != 0
    assert "nv12 frames need an even height and width" in lib.anakin_last_error().decode()


# ---------------------------------------------------------------------------------------------- Worker
def _worker_graph(batch, filt="pil", name="nv12", max_hw=(96, 96)):
    from anakin_b200 import anakin_bin, api, modelzoo
    G = api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build("tiny_resnet", batch=batch, precision="int8")))
    G.set_input_image("input_0", MEAN[:3], SCALE[:3], [0, 1, 2])
    G.set_input_image_resize("input_0", max_hw[0], max_hw[1], 36, filter=filt, pixel_format=name)
    G.ResetBatchSize("input_0", batch)
    return G


def _net_rows(net, frames, boxes):
    net.set_input_crops("input_0", frames, boxes)
    net.prediction(); net.sync()
    return net.read_tensor(net.out_names[0])[0].reshape(len(boxes), -1).copy()


def test_worker_sync_and_async_crops_requests_match_a_single_net():
    import torch
    from anakin_b200 import api
    batch = 2
    G = _worker_graph(batch)
    f = [Y.random_frame(h, w, Y.NV12, 60 + i) for i, (h, w) in enumerate([(96, 96), (40, 76), (2, 2), (90, 6)])]
    reqs = [([f[0]], [(0, 1, 3, 5, 7), (0, 0, 0, 96, 96)]), ([f[1], f[2]], [(1, 0, 0, 2, 2), (0, 3, 3, 37, 73)]),
            ([f[3]], [(0, 5, 1, 80, 5), (0, 0, 0, 1, 1)]), ([f[0], f[3]], [(1, 0, 0, 90, 6), (0, 31, 17, 33, 61)])]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tiny_nv12.anakin.bin")
        G.save(path)
        G.Optimize()
        net = api.Net(G, "int8")
        want = [_net_rows(net, fr, bx).reshape(-1) for fr, bx in reqs]
        w = api.Worker(path, "int8", threads=2)
        w.wait_ready()
        packed = [api.pack_images(fr) + (api.pack_boxes(bx),) for fr, bx in reqs]
        pins = [tuple(torch.from_numpy(a).pin_memory() for a in p) for p in packed]
        outs = [torch.empty(want[0].size, dtype=torch.float32).pin_memory() for _ in reqs]
        for _ in range(2):      # the second round replays each thread's captured graph
            for (p, h, b), o in zip(pins, outs):
                w.async_prediction_crops_ptr(p.data_ptr(), p.numel(), h.data_ptr(), h.shape[0], b.data_ptr(),
                                             b.shape[0], o.data_ptr(), o.numel())
            for _ in reqs:
                w.async_get_result()
            for i, (o, ref) in enumerate(zip(outs, want)):
                assert np.array_equal(o.numpy(), ref), i
            for (fr, bx), ref in zip(reqs, want):
                assert np.array_equal(w.sync_prediction_crops(fr, bx, ref.size), ref)
        # without a batching window a request carries the whole batch
        with pytest.raises(api.AnakinError, match="1 boxes, the batch is 2"):
            w.sync_prediction_crops([f[0]], [(0, 0, 0, 4, 4)], want[0].size)
        del w


def test_batching_worker_gathers_crops_and_images_and_malformed_requests_fail_alone():
    import torch
    from anakin_b200 import api
    batch = 4
    G = _worker_graph(batch, filt="reference")
    f = [Y.random_frame(h, w, Y.NV12, 80 + i) for i, (h, w) in enumerate([(96, 96), (40, 76), (2, 2), (90, 6)])]
    rA = ([f[0]], [(0, 3, 1, 81, 93)])
    rB = ([f[1], f[2]], [(1, 0, 1, 2, 1), (0, 1, 1, 39, 75)])
    rC = [f[3]]                                                       # an images request
    bad_box = ([f[1]], [(0, 1, 0, 40, 76)])                           # one row past the frame
    bad_frame = ([f[2]], [(1, 0, 0, 1, 1)])                           # no frame 1
    bad_count = ([f[0], f[1]], [(0, 0, 0, 1, 1)])                     # 2 frames for 1 box
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tiny_nv12.anakin.bin")
        G.save(path)
        G.Optimize()
        net = api.Net(G, "int8")
        want = _net_rows(net, [f[0], f[1], f[2], f[3]], [(0, 3, 1, 81, 93), (2, 0, 1, 2, 1), (1, 1, 1, 39, 75),
                                                         (3, 0, 0, 90, 6)])
        # a 0.1 s window: the requests below are queued long before it closes, so they are gathered
        w = api.Worker(path, "int8", threads=1, devices=(0,), max_delay_us=100000)
        out0 = w.image_sizes()["output"]
        order = [rA, bad_box, rB, bad_frame, rC, bad_count]
        pins = []
        for r in order:
            if isinstance(r, tuple):
                pix, hw = api.pack_images(r[0])
                bx = api.pack_boxes(r[1])
            else:
                (pix, hw), bx = api.pack_images(r), None
            k = len(r[1]) if bx is not None else len(r)
            pins.append([torch.from_numpy(a).pin_memory() for a in ((pix, hw) if bx is None else (pix, hw, bx))]
                        + [torch.zeros(k * out0, dtype=torch.float32).pin_memory()])
        for r, p in zip(order, pins):
            if len(p) == 4:
                w.async_prediction_crops_ptr(p[0].data_ptr(), p[0].numel(), p[1].data_ptr(), p[1].shape[0],
                                             p[2].data_ptr(), p[2].shape[0], p[3].data_ptr(), p[3].numel())
            else:
                w.async_prediction_images_ptr(p[0].data_ptr(), p[0].numel(), p[1].data_ptr(), p[1].shape[0],
                                              p[2].data_ptr(), p[2].numel())
        w.async_get_result()
        with pytest.raises(api.AnakinError, match=r"box 0 \(frame 0, top 1, left 0, 40 x 76\) is not inside frame 0"):
            w.async_get_result()
        w.async_get_result()
        with pytest.raises(api.AnakinError, match="no frame 1 among the request's 1"):
            w.async_get_result()
        w.async_get_result()
        with pytest.raises(api.AnakinError, match="2 frames for 1 boxes"):
            w.async_get_result()
        got = [p[-1].numpy() for p in pins]
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[1:3].reshape(-1))
        assert np.array_equal(got[4], want[3])
        assert not got[1].any() and not got[3].any() and not got[5].any()
        predictions, images = w.batch_stats()
        del w
    assert predictions >= 1 and images == 4
