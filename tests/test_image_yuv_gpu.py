"""GPU: NV12 / I420 frames as resizing image inputs (b200_image_resize_yuv_run, b200_image_resize_pil_yuv_run, the
`<input>:ImageResize` op with image_pixel_format 1 / 2). Every comparison is bit for bit, with deterministic seeds: the
kernels against the composed numpy restatement (tests/yuv_oracle.py, pinned to OpenCV and Pillow by
tests/test_cpu_image_yuv.py), and a YUV Net against the interleaved resize Net fed the restated RGB of the same
frames."""
import ctypes as C
import os
import tempfile
import zlib

import numpy as np
import pytest

import yuv_oracle as Y

pytestmark = pytest.mark.gpu

MEAN = [123.675, 116.28, 103.53]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375]
FILTERS = {"reference": 0, "pil": 1}


def _frames(sizes, fmt, seed):
    return [Y.random_frame(h, w, fmt, seed * 1000 + i) for i, (h, w) in enumerate(sizes)]


# ---------------------------------------------------------------------------------------------- 1. kernels
def _run_kernel(frames, fmt, filt, s, oh, ow, max_hw):
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
        off += h * w * 3 // 2
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = len(frames), 3, oh, ow
    src = torch.from_numpy(pix).cuda()
    tab = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).cuda()
    out = torch.full((len(frames), oh, ow, 3), 7, dtype=torch.uint8, device="cuda")
    if filt == "pil":
        nbytes = C.c_size_t()
        A.check(lib.b200_image_resize_pil_workspace(C.byref(d), max_hw[0], max_hw[1], s, C.byref(nbytes)), "workspace")
        ws = torch.full((nbytes.value,), 0xA5, dtype=torch.uint8, device="cuda")
        A.check(lib.b200_image_resize_pil_yuv_run(C.byref(d), fmt, max_hw[0], max_hw[1], s, ptr(src), ptr(tab), ptr(ws),
                                                  ptr(out), stream_ptr()), "image_resize_pil_yuv")
    else:
        A.check(lib.b200_image_resize_yuv_run(C.byref(d), fmt, ptr(src), ptr(tab), ptr(out), stream_ptr()),
                "image_resize_yuv")
    torch.cuda.synchronize()
    return out.cpu().numpy()


# identity, 2x down, 1080p and 720p both ways, an upscale, the smallest frame, an extreme aspect, and Pillow's
# pass-order cases on both sides of the switch
KERNEL_SOURCES = [(224, 224), (448, 448), (1080, 1920), (1920, 1080), (720, 1280), (100, 150), (2, 2), (16, 1000),
                  (2000, 16), (1600, 16)]


@pytest.mark.parametrize("net_hw", [(224, 224), (200, 160)])
@pytest.mark.parametrize("s", [0, 232, 256])
@pytest.mark.parametrize("filt", ["reference", "pil"])
@pytest.mark.parametrize("name", ["nv12", "i420"])
def test_kernel_equals_composed_restatement(name, filt, s, net_hw):
    fmt = Y.FORMATS[name]
    oh, ow = net_hw
    frames = _frames(KERNEL_SOURCES, fmt, zlib.crc32(repr((name, filt, s, net_hw)).encode()))
    max_hw = (max(h for h, _ in KERNEL_SOURCES), max(w for _, w in KERNEL_SOURCES))
    widths = [ow] + ([222] if net_hw == (224, 224) else [])     # 222: the byte-store instance
    for w_out in widths:
        got = _run_kernel(frames, fmt, filt, s, oh, w_out, max_hw)
        for i, f in enumerate(frames):
            want = Y.resize(f, fmt, filt, s, oh, w_out)
            assert np.array_equal(got[i], want), (KERNEL_SOURCES[i], w_out, int(np.abs(got[i].astype(int) - want).max()))


# ---------------------------------------------------------------------------------------------- 2. every triple
@pytest.mark.parametrize("filt", ["reference", "pil"])
@pytest.mark.parametrize("name", ["nv12", "i420"])
def test_identity_stretch_converts_every_triple(name, filt):
    """Both filters are the identity at scale 1, so a 4096 x 4096 stretch to itself is the conversion alone."""
    fmt = Y.FORMATS[name]
    frame = Y.exhaustive_frame(fmt)
    n = Y.EXHAUSTIVE
    got = _run_kernel([frame], fmt, filt, 0, n, n, (n, n))[0]
    assert np.array_equal(got, Y.yuv_to_rgb(frame, fmt))


# ---------------------------------------------------------------------------------------------- 3. Net
def _graphs(g_dict, batch, max_hw, resize_short, filt, name):
    """(interleaved resize Graph, YUV resize Graph) from one model dict."""
    from anakin_b200 import anakin_bin, api
    blob = anakin_bin.dumps(g_dict)
    Gi, Gy = api.Graph.from_bytes(blob), api.Graph.from_bytes(blob)
    for G, pf in ((Gi, "interleaved"), (Gy, name)):
        G.set_input_image("input_0", MEAN, SCALE, [0, 1, 2])
        G.set_input_image_resize("input_0", max_hw[0], max_hw[1], resize_short, filter=filt, pixel_format=pf)
        G.ResetBatchSize("input_0", batch)
        G.Optimize()
    return Gi, Gy


def compare_nets(model, precision, batch, resize_short, size_sets, max_hw, filt, name, exports=None,
                 check_graph=False):
    """A YUV Net and the interleaved resize Net fed the restated RGB: same outputs and exports bit for bit, the same
    launches, and the YUV Net's input tensor holds the composed restatement, for every request in size_sets."""
    from anakin_b200 import api, modelzoo, saber_abi
    fmt = Y.FORMATS[name]
    g_dict = modelzoo.build(model, batch=batch, precision=precision)
    shape = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"]
    H, W = shape[2], shape[3]
    Gi, Gy = _graphs(g_dict, batch, max_hw, resize_short, filt, name)
    ni, ny = api.Net(Gi, precision, exports=exports), api.Net(Gy, precision, exports=exports)
    assert ny.exec_order() == ni.exec_order() and ny.launched_ops() == ni.launched_ops()
    lib = saber_abi.load()
    for it, sizes in enumerate(size_sets):
        frames = _frames(sizes, fmt, seed=100 * it + batch)
        ni.set_input_images("input_0", [Y.yuv_to_rgb(f, fmt) for f in frames])
        ny.set_input_images("input_0", frames)
        n0 = lib.b200_launch_count()
        ny.prediction()
        n1 = lib.b200_launch_count()
        ni.prediction()
        n2 = lib.b200_launch_count()
        ni.sync(); ny.sync()
        assert n1 - n0 == n2 - n1, (n1 - n0, n2 - n1)
        if check_graph and it >= 2:
            assert ny.cuda_graph_active() and n1 == n0, (it, n1 - n0)
        want_in = Y.resize_batch(frames, fmt, filt, resize_short, H, W)
        assert np.array_equal(ny.read_tensor("input_0")[0], want_in), (model, precision, it)
        for nm in ni.out_names:
            assert np.array_equal(ni.get_output(nm).view(np.uint8), ny.get_output(nm).view(np.uint8)), (nm, it)
        for x in exports or []:
            assert np.array_equal(ni.get_export(x).view(np.uint32), ny.get_export(x).view(np.uint32)), (x, it)
    assert ny.cuda_graph_active()
    return ny


TINY_SETS = [[(32, 32), (76, 42)], [(2, 2), (80, 96)], [(34, 64), (96, 18)]]


@pytest.mark.parametrize("precision", ["fp32", "fp16", "int8"])
@pytest.mark.parametrize("model", ["tiny_resnet", "tiny_mobilenet"])
def test_tiny_nets_equal_the_interleaved_net(model, precision):
    for i, (filt, name) in enumerate([("reference", "nv12"), ("pil", "i420")]):
        compare_nets(model, precision, 2, 36, TINY_SETS[i:] + TINY_SETS[:i], (96, 96), filt, name)


def test_resnet50_int8_1080p_pil_equals_the_interleaved_net():
    sets = [[(1080, 1920)] * 8, [(1080, 1920), (1920, 1080), (720, 1280), (1080, 1440)] * 2]
    compare_nets("resnet50", "int8", 8, 256, sets, (1920, 1920), "pil", "nv12", exports=["pool5"])


# ---------------------------------------------------------------------------------------------- 4. CUDA graph
@pytest.mark.parametrize("filt", ["reference", "pil"])
def test_cuda_graph_serves_frames_of_different_sizes(filt):
    sets = [[(32, 32), (76, 42)], [(600, 600), (2, 2)], [(40, 600), (600, 42)], [(96, 96), (590, 6)],
            [(18, 90), (64, 34)], [(600, 300), (300, 600)]]
    compare_nets("tiny_resnet", "int8", 2, 36, sets, (600, 600), filt, "i420", check_graph=True)


# ---------------------------------------------------------------------------------------------- 5. Worker
def _yuv_graph(batch, max_hw=(96, 96), name="nv12", filt="reference"):
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build("tiny_resnet", batch=batch, precision="int8")
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.set_input_image("input_0", MEAN, SCALE, [0, 1, 2])
    G.set_input_image_resize("input_0", max_hw[0], max_hw[1], 36, filter=filt, pixel_format=name)
    G.ResetBatchSize("input_0", batch)
    return G


def _net_rows(net, frames):
    net.set_input_images("input_0", frames)
    net.prediction(); net.sync()
    return net.read_tensor(net.out_names[0])[0].reshape(len(frames), -1).copy()


def test_worker_sync_and_async_nv12_requests_match_a_single_net():
    import torch
    from anakin_b200 import api
    batch = 2
    G = _yuv_graph(batch, (600, 600), filt="pil")
    size_sets = [[(32, 32), (76, 42)], [(2, 2), (600, 96)], [(34, 64), (96, 18)], [(600, 600), (50, 50)],
                 [(590, 6), (64, 34)], [(40, 40), (42, 38)]]
    reqs = [_frames(s, Y.NV12, seed=i) for i, s in enumerate(size_sets)]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tiny_nv12.anakin.bin")
        G.save(path)
        G.Optimize()
        net = api.Net(G, "int8")
        want = [_net_rows(net, f).reshape(-1) for f in reqs]
        w = api.Worker(path, "int8", threads=2)
        w.wait_ready()
        packed = [api.pack_images(f) for f in reqs]
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
        assert np.array_equal(w.sync_prediction_images(reqs[3], want[3].size), want[3])
        del w


def test_batching_worker_gathers_frames_and_a_malformed_frame_fails_alone():
    import torch
    from anakin_b200 import api
    batch = 4
    G = _yuv_graph(batch)
    frames = _frames([(32, 32), (76, 42), (96, 96), (2, 2)], Y.NV12, seed=9)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tiny_nv12.anakin.bin")
        G.save(path)
        G.Optimize()
        net = api.Net(G, "int8")
        want = _net_rows(net, frames)
        # a 0.1 s window: the requests below are queued long before it closes, so they are gathered
        w = api.Worker(path, "int8", threads=1, devices=(0,), max_delay_us=100000)
        out0 = w.image_sizes()["output"]
        odd = np.zeros((33 * 3 // 2, 32), np.uint8)                        # a 33 x 32 frame: odd height
        short = frames[1][:-1]                                             # 76 x 42 less a chroma row
        reqs = [[frames[0]], [odd], [frames[1]], [frames[2]], [short], [frames[3]]]
        pins = []
        for r in reqs:
            pix = np.concatenate([f.reshape(-1) for f in r])
            hw = np.array([[33, 32]] if r[0] is odd else [[f.shape[0] * 2 // 3, f.shape[1]] for f in r], np.int32)
            if r[0] is short:
                hw = np.array([[76, 42]], np.int32)
            pins.append((torch.from_numpy(pix).pin_memory(), torch.from_numpy(hw).pin_memory(),
                         torch.zeros(out0, dtype=torch.float32).pin_memory()))
        for p, h, o in pins:
            w.async_prediction_images_ptr(p.data_ptr(), p.numel(), h.data_ptr(), h.shape[0], o.data_ptr(), o.numel())
        w.async_get_result()
        with pytest.raises(api.AnakinError, match="nv12 frames need an even height and width"):
            w.async_get_result()
        w.async_get_result()
        w.async_get_result()
        with pytest.raises(api.AnakinError, match="pixel bytes, the sizes need %d" % (76 * 42 * 3 // 2)):
            w.async_get_result()
        w.async_get_result()
        got = [o.numpy() for _, _, o in pins]
        for i, j in ((0, 0), (2, 1), (3, 2), (5, 3)):
            assert np.array_equal(got[i], want[j]), (i, j)
        assert not got[1].any() and not got[4].any()
        stats = w.batch_stats()
        assert np.array_equal(w.sync_prediction_images([frames[2]], out0), want[2])
        del w
    assert stats


# ---------------------------------------------------------------------------------------------- 6. refusals
def test_net_refuses_a_yuv_format_without_resize_or_three_channels():
    from anakin_b200 import anakin_bin, api
    G = _yuv_graph(2)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        with open(p, "rb") as f:
            gd = anakin_bin.loads(f.read())
    attrs = gd["nodes"][[n["op"] for n in gd["nodes"]].index("Input")]["attrs"]
    for k in ("image_max_h", "image_max_w", "image_resize_short", "image_resize_filter"):
        attrs.pop(k)
    G2 = api.Graph.from_bytes(anakin_bin.dumps(gd))
    G2.Optimize()
    with pytest.raises(api.AnakinError, match="input input_0: image_pixel_format 1 needs an image input with "
                                              "on-device resize"):
        api.Net(G2, "int8")
    G1 = api.Graph.from_bytes(anakin_bin.dumps(gd))
    G1.Reshape("input_0", [2, 1] + G1.input_shape("input_0")[2:])
    G1.set_input_image("input_0", MEAN[:1], SCALE[:1], [0])
    G1.set_input_image_resize("input_0", 96, 96, 36, pixel_format="i420")
    G1.Optimize()
    with pytest.raises(api.AnakinError, match="input input_0: i420 frames need 3 channels"):
        api.Net(G1, "fp32")
