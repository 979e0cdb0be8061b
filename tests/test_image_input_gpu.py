"""GPU: 8-bit image graph inputs (uint8 HWC pixels normalised inside the first convolution) against the fp32 input fed
the host-normalised tensor. Every comparison is bit for bit: the normalisation ((u - mean) * scale, two fp32 roundings,
no FMA) is what numpy computes in float32, and everything after it is the fp32 input's path.

Every case uses a non-zero mean and padded convolutions; the INT8 cases use a scale that drives some inputs past the
quantisation clamp."""
import ctypes as C
import os
import tempfile
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# ImageNet-style normalisation of 8-bit pixels: x in about [-2.1, 2.6]
MEAN = [123.675, 116.28, 103.53, 64.0]
SCALE = [1 / 58.395, 1 / 57.12, 1 / 57.375, 1 / 40.0]


def normalise(u8_nhwc, mean, scale, src):
    """The host-normalised fp32 NCHW tensor an image input stands for (numpy float32 arithmetic)."""
    c = u8_nhwc.shape[-1]
    u = u8_nhwc[..., list(src)].astype(np.float32)
    x = (u - np.asarray(mean[:c], np.float32)) * np.asarray(scale[:c], np.float32)
    assert x.dtype == np.float32
    return np.ascontiguousarray(x.transpose(0, 3, 1, 2))


def _order(c, swap):
    if not swap or c == 1:
        return list(range(c))
    return [2, 1, 0] if c == 3 else [2, 1, 0, 3][:c] if c == 4 else list(range(c))[::-1]


# ---------------------------------------------------------------------------------------------- 1. stem kernel
# (n, c, h, w, k, r, s, stride, pad, pool) ; pool = None | (window, stride, pad)
STEM_CASES = [
    (2, 3, 224, 224, 64, 7, 7, 2, 3, (3, 2, 0)),     # ResNet-50 conv1 + pool1
    (2, 3, 64, 64, 32, 3, 3, 2, 1, None),            # MobileNet conv1
    (1, 3, 48, 40, 64, 3, 3, 1, 1, (2, 2, 0)),       # VGG16 3x3/s1 + 2x2/s2 pool
    (3, 3, 37, 45, 64, 7, 7, 2, 3, (3, 2, 0)),       # ragged
    (2, 1, 30, 30, 48, 3, 3, 1, 1, (2, 2, 0)),       # one channel
    (1, 4, 20, 28, 128, 3, 3, 1, 1, None),           # four channels, two n-tiles
]
KINDS = ["i8_u8", "i8_s8", "i8_f32", "f16", "tf32x3"]


def _stem_desc(A, math, out_dtype, case, ldc, inv_scale):
    n, c, h, w, k, r, s, stride, pad, pool = case
    d = A.StemDesc()
    d.math, d.out_dtype = math, out_dtype
    d.n, d.c, d.h, d.w, d.k, d.ldc = n, c, h, w, k, ldc
    d.r, d.s, d.stride_h, d.stride_w, d.pad_h, d.pad_w = r, s, stride, stride, pad, pad
    d.relu, d.neg_slope, d.in_inv_scale = 1, 0.0, inv_scale
    d.monotone_epilogue = 1
    if pool is not None:
        d.fuse_pool, d.pool_type = 1, A.POOL_MAX
        d.pool_window_h = d.pool_window_w = pool[0]
        d.pool_stride_h = d.pool_stride_w = pool[1]
        d.pool_pad_h = d.pool_pad_w = pool[2]
    return d


@pytest.mark.parametrize("swap", [False, True])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", STEM_CASES)
def test_stem_image_equals_stem_on_normalised_input(case, kind, swap):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    lib = A.load()
    n, c, h, w, k, r, s, stride, pad, pool = case
    rng = np.random.default_rng(zlib.crc32(repr((case, kind, swap)).encode()))
    u8 = rng.integers(0, 256, (n, h, w, c), dtype=np.uint8)
    src = _order(c, swap)
    x = normalise(u8, MEAN, SCALE, src)
    math, out_dtype = {"i8_u8": (A.MATH_I8, A.UINT8), "i8_s8": (A.MATH_I8, A.INT8), "i8_f32": (A.MATH_I8, A.FLOAT),
                       "f16": (A.MATH_F16, A.HALF), "tf32x3": (A.MATH_TF32X3, A.FLOAT)}[kind]
    es = {A.UINT8: 1, A.INT8: 1, A.HALF: 2, A.FLOAT: 4}[out_dtype]
    ldc = (k * es + 15) // 16 * 16 // es
    inv_scale = float(np.float32(127.0 / 1.5))       # |x| > 1.5 saturates
    bias = rng.uniform(-0.5, 0.5, k).astype(np.float32)
    scale = None
    if math == A.MATH_I8:
        wt = rng.integers(-127, 128, (k, c, r, s)).astype(np.int8)
        bias = rng.uniform(-2000, 2000, k).astype(np.float32)
        scale = rng.uniform(0.5, 1.5, k).astype(np.float32) * np.float32(1.0 / (40.0 * np.sqrt(c * r * s) * 8))
    elif math == A.MATH_F16:
        wt = (rng.standard_normal((k, c, r, s)) * 0.2).astype(np.float16)
    else:
        wt = (rng.standard_normal((k, c, r, s)) * 0.2).astype(np.float32)
    d = _stem_desc(A, math, out_dtype, case, ldc, inv_scale if math == A.MATH_I8 else 1.0)
    oh, ow = C.c_int32(), C.c_int32()
    A.check(lib.b200_stem_conv_out_hw(C.byref(d), C.byref(oh), C.byref(ow)), "stem_out_hw")
    packed = np.zeros(lib.b200_stem_packed_weight_bytes(C.byref(d)), np.uint8)
    A.check(lib.b200_stem_pack_weights(C.byref(d), np.ascontiguousarray(wt).ctypes.data_as(C.c_void_p),
                                       packed.ctypes.data_as(C.c_void_p)), "stem_pack")
    wd, bd = dev(packed), dev(bias)
    sd = dev(scale) if scale is not None else None
    tdt = {A.UINT8: torch.uint8, A.INT8: torch.int8, A.HALF: torch.float16, A.FLOAT: torch.float32}[out_dtype]
    want = torch.full((n, oh.value, ow.value, ldc), 7, dtype=tdt, device="cuda")
    got = torch.full((n, oh.value, ow.value, ldc), 7, dtype=tdt, device="cuda")
    A.check(lib.b200_stem_conv_run(C.byref(d), ptr(dev(x)), ptr(wd), ptr(bd), ptr(sd), ptr(want), stream_ptr()), "fp32")
    fmt = A.image_desc(MEAN[:c], SCALE[:c], src)
    A.check(lib.b200_stem_conv_run_image(C.byref(d), C.byref(fmt), ptr(dev(u8)), ptr(wd), ptr(bd), ptr(sd), ptr(got),
                                         stream_ptr()), "image")
    torch.cuda.synchronize()
    want, got = want.cpu().numpy(), got.cpu().numpy()
    if math == A.MATH_I8 and out_dtype != A.FLOAT:
        assert (np.abs(x) * inv_scale > 127).any(), "the case must drive inputs past the clamp"
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))


# ---------------------------------------------------------------------------------------------- 2. layout transform
@pytest.mark.parametrize("extra", [0, 16, -1])     # bytes past the 16-byte-rounded pixel; -1: c_pad = c
@pytest.mark.parametrize("dtype", ["f32", "f16", "s8", "u8"])
@pytest.mark.parametrize("c", [1, 3, 4])
def test_image_to_nhwc_equals_nchw_to_nhwc(c, dtype, extra):
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import dev, ptr, stream_ptr
    lib = A.load()
    out_dtype, es, tdt = {"f32": (A.FLOAT, 4, torch.float32), "f16": (A.HALF, 2, torch.float16),
                          "s8": (A.INT8, 1, torch.int8), "u8": (A.UINT8, 1, torch.uint8)}[dtype]
    c_pad = c if extra < 0 else ((c * es + 15) // 16 * 16 + extra) // es
    n, h, w = 2, 19, 23
    rng = np.random.default_rng(c * 100 + es * 10 + extra)
    u8 = rng.integers(0, 256, (n, h, w, c), dtype=np.uint8)
    for swap in (False, True):
        src = _order(c, swap)
        x = normalise(u8, MEAN, SCALE, src)
        inv_scale = float(np.float32(127.0 / 1.5))
        want = torch.full((n, h, w, c_pad), 5, dtype=tdt, device="cuda")
        got = torch.full((n, h, w, c_pad), 5, dtype=tdt, device="cuda")
        A.check(lib.b200_nchw_to_nhwc(ptr(dev(x)), ptr(want), out_dtype, n, c, h, w, c_pad, inv_scale, stream_ptr()), "ref")
        fmt = A.image_desc(MEAN[:c], SCALE[:c], src)
        A.check(lib.b200_image_to_nhwc(C.byref(fmt), ptr(dev(u8)), ptr(got), out_dtype, n, c, h, w, c_pad, inv_scale,
                                       stream_ptr()), "image")
        torch.cuda.synchronize()
        assert np.array_equal(got.cpu().numpy().view(np.uint8), want.cpu().numpy().view(np.uint8)), (c, dtype, extra, swap)


# ---------------------------------------------------------------------------------------------- 3.-6. Net / Worker
FMT_SRC = [2, 1, 0]     # BGR pixels, RGB network


def _graphs(g_dict, batch):
    """(fp32-input Graph, image-input Graph) from one model dict."""
    from anakin_b200 import anakin_bin, api
    blob = anakin_bin.dumps(g_dict)
    Gf, Gi = api.Graph.from_bytes(blob), api.Graph.from_bytes(blob)
    c = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"][1]
    Gi.set_input_image("input_0", MEAN[:c], SCALE[:c], _order(c, True))
    for G in (Gf, Gi):
        G.ResetBatchSize("input_0", batch)
        G.Optimize()
    return Gf, Gi


def _images(batch, h, w, c, seed=3):
    return np.random.default_rng(seed).integers(0, 256, (batch, h, w, c), dtype=np.uint8)


def compare_nets(model, precision, batch, hw=None, g_dict=None):
    """Build the model twice (fp32 input / image input), run both on the same images and compare every output bit for
    bit, eager and CUDA-graph replay; returns the image Net."""
    from anakin_b200 import api, modelzoo
    if g_dict is None:
        g_dict = modelzoo.build(model, batch=batch, precision=precision)
    shape = next(n for n in g_dict["nodes"] if n["op"] == "Input")["attrs"]["input_shape"]
    c, h, w = shape[1], shape[2], shape[3]
    Gf, Gi = _graphs(g_dict, batch)
    u8 = _images(batch, h, w, c)
    x = normalise(u8, MEAN, SCALE, _order(c, True))
    nf, ni = api.Net(Gf, precision), api.Net(Gi, precision)
    info = ni.tensor_info("input_0")
    assert (info["dtype"], info["layout"], info["c_stored"], info["bytes"]) == (7, 9, c, u8.nbytes), info
    assert nf.launched_ops() == ni.launched_ops(), "the normalisation must not cost a launch"
    nf.set_input("input_0", x)
    ni.set_input_image("input_0", u8)
    first = {}
    for it in range(3):                 # eager, then captured CUDA graph, then replay
        nf.prediction(); ni.prediction(); nf.sync(); ni.sync()
        for name in nf.out_names:
            a, b = nf.get_output(name), ni.get_output(name)
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (model, precision, name, it)
            first.setdefault(name, b)
            assert np.array_equal(b.view(np.uint8), first[name].view(np.uint8)), ("replay differs", name, it)
    assert ni.cuda_graph_active()
    return ni


@pytest.mark.parametrize("precision", ["fp32", "fp16", "int8"])
@pytest.mark.parametrize("model", ["tiny_resnet", "tiny_mobilenet"])
def test_tiny_nets_image_input_bit_exact(model, precision):
    compare_nets(model, precision, 2)


@pytest.mark.parametrize("model,precision,batch", [("resnet50", "int8", 8), ("resnet50", "fp32", 1),
                                                   ("mobilenet_v1", "fp16", 16), ("vgg16", "fp32", 1)])
def test_benchmark_nets_image_input_bit_exact(model, precision, batch):
    compare_nets(model, precision, batch)


def dilated_tiny_resnet(batch, precision):
    """tiny_resnet with conv1 dilated by 2 (padding 6 keeps its output size): the fused stem refuses a dilated filter, so
    the graph input goes through the NHWC transform (b200_nchw_to_nhwc / b200_image_to_nhwc) and the R x S conv plan,
    with the MAX pooling in a launch of its own. The INT8 calibration table still applies by edge name."""
    from anakin_b200 import modelzoo
    g = modelzoo.build("tiny_resnet", batch=batch, precision=precision)
    attrs = next(n for n in g["nodes"] if n["name"] == "conv1")["attrs"]
    attrs["dilation_rate"], attrs["padding"] = [2, 2], [6, 6]
    return g


def eager_launches(net):
    """Kernel launches of one eager prediction of `net`, which keeps its staged input."""
    from anakin_b200 import saber_abi
    lib = saber_abi.load()
    net.set_cuda_graph(False)
    n0 = lib.b200_launch_count()
    net.prediction()
    net.sync()
    return lib.b200_launch_count() - n0


@pytest.mark.parametrize("precision", ["fp32", "fp16", "int8"])
def test_transform_path_bit_exact_without_fused_stem(precision):
    """A first conv the fused stem refuses: both Nets convert their input in a separate transform and run the same
    R x S conv plan -- bit-exact at every precision. The transform and the pooling after the conv are two launches more
    than the stem-fused twin's single one."""
    ni = compare_nets(None, precision, 2, g_dict=dilated_tiny_resnet(2, precision))
    twin = compare_nets("tiny_resnet", precision, 2)
    assert eager_launches(ni) == eager_launches(twin) + 2


def _small_graph(kind):
    from anakin_b200 import modelzoo
    b = modelzoo.GraphBuilder("img_" + kind, seed=5)
    x = b.input("input_0", (2, 3, 20, 24))
    if kind == "conv1x1":             # no fused stem: the transform path
        y = b.conv("conv1", x, 3, 32, 1, 1, 0, bias=True)
        y = b.relu("relu1", y)
        y = b.conv("conv2", y, 32, 16, 3, 1, 1, bias=True)
        b.output("out", y)
    elif kind == "two_convs":         # one image input read by two convolutions
        y = b.conv("conv_a", x, 3, 16, 3, 1, 1, bias=True)
        z = b.conv("conv_b", x, 3, 16, 5, 2, 2, bias=True)
        b.output("out_a", y)
        b.output("out_b", z)
    elif kind == "pool_after":        # both ways a MAX pooling ends up in its own launch after the conv
        y = b.conv("conv1", x, 3, 16, 3, 1, 1, bias=True)    # fused stem; a 12 x 12 window is too large for its pooling
        y = b.relu("relu1", y)
        y = b.pool("pool1", y, 12, 4)
        y = b.conv("conv2", y, 16, 32, 1, 1, 0, bias=True)   # no conv plan fuses a pooling behind a 1 x 1 filter
        y = b.relu("relu2", y)
        y = b.pool("pool2", y, 2, 2)
        b.output("out", y)
    elif kind == "stem_refused":      # stride 5: the fused stem refuses it, both inputs take the transform path
        y = b.conv("conv1", x, 3, 16, 5, 5, 0, bias=True)
        y = b.relu("relu1", y)
        b.output("out", y)
    else:                             # a Pooling reads the image
        y = b.conv("conv1", x, 3, 16, 3, 1, 1, bias=True)
        z = b.pool("pool_in", x, 2, 2)
        b.output("out_a", y)
        b.output("out_b", z)
    return b.finalize()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("kind", ["conv1x1", "two_convs", "pool_after", "stem_refused"])
def test_builder_graphs_bit_exact(kind, precision):
    compare_nets(None, precision, 2, g_dict=_small_graph(kind))


def test_image_input_read_by_pooling_fails_init_naming_the_consumer():
    from anakin_b200 import api
    _, Gi = _graphs(_small_graph("pool"), 2)
    with pytest.raises(api.AnakinError, match=r"image input input_0 is read by node pool_in \(op Pooling\)"):
        api.Net(Gi, "fp32")


def test_input_kind_mismatch_fails():
    from anakin_b200 import api, modelzoo
    Gf, Gi = _graphs(modelzoo.build("tiny_resnet", 2), 2)
    nf, ni = api.Net(Gf, "fp32"), api.Net(Gi, "fp32")
    u8 = _images(2, 32, 32, 3)
    # n*h*w*3 bytes == count*4 floats when the float count is a quarter: the marker decides, not the size
    with pytest.raises(api.AnakinError, match="image input"):
        ni.set_input_ptr("input_0", u8.ctypes.data, u8.nbytes // 4)
    with pytest.raises(api.AnakinError, match="not an image input"):
        nf.set_input_image("input_0", np.zeros((2, 32, 32, 3 * 4), np.uint8))
    with pytest.raises(api.AnakinError):
        ni.set_input_image("input_0", u8[:1])


def test_worker_async_image_requests_match_a_single_net():
    import torch
    from anakin_b200 import anakin_bin, api, modelzoo
    batch = 2
    g = modelzoo.build("tiny_resnet", batch=batch, precision="int8")
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    G.set_input_image("input_0", MEAN[:3], SCALE[:3], FMT_SRC)
    reqs = [_images(batch, 32, 32, 3, seed=s) for s in range(6)]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "tiny_image.anakin.bin")
        G.save(path)
        G.Optimize()
        net = api.Net(G, "int8")
        want = []       # the Worker returns the output's raw storage (NHWC, channels padded)
        for u8 in reqs:
            net.set_input_image("input_0", u8)
            net.prediction(); net.sync()
            want.append(net.read_tensor(net.out_names[0])[0].reshape(-1).copy())
        w = api.Worker(path, "int8", threads=2)
        w.wait_ready()
        ins = [torch.from_numpy(u).pin_memory() for u in reqs]
        outs = [torch.empty(want[0].size, dtype=torch.float32).pin_memory() for _ in reqs]
        for i, o in zip(ins, outs):
            w.async_prediction_image_ptr(i.data_ptr(), i.numel(), o.data_ptr(), o.numel())
        for _ in reqs:
            w.async_get_result()
        for o, ref in zip(outs, want):
            assert np.array_equal(o.numpy(), ref)
        got = w.sync_prediction_image(reqs[0], want[0].size)
        assert np.array_equal(got, want[0])
        # a request one byte short or long fails alone, as Net.set_input_image would; the one queued after it is served
        for n in (ins[0].numel() - 1, ins[0].numel() + 1):
            outs[1].zero_()
            w.async_prediction_image_ptr(ins[0].data_ptr(), n, outs[0].data_ptr(), outs[0].numel())
            w.async_prediction_image_ptr(ins[1].data_ptr(), ins[1].numel(), outs[1].data_ptr(), outs[1].numel())
            with pytest.raises(api.AnakinError, match="image of %d bytes, input input_0 holds %d" % (n, ins[0].numel())):
                w.async_get_result()
            w.async_get_result()
            assert np.array_equal(outs[1].numpy(), want[1])
        # the float calls fail on an image input
        with pytest.raises(api.AnakinError, match="image input"):
            w.sync_prediction(np.zeros((batch, 3, 32, 32), np.float32), want[0].size)
        del w
