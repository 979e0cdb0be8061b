"""8-bit image graph inputs without a GPU: the Graph API that declares them (stored on the Input node, kept by save /
load and ResetBatchSize), its rejections, and the argument checks of the two kernels' entry points, which run before
the device check."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

FMT = {"mean": [123.675, 116.28, 103.53], "scale": [1 / 58.395, 1 / 57.12, 1 / 57.375], "src_channel": [2, 1, 0]}


def _graph(model="tiny_resnet"):
    from anakin_b200 import anakin_bin, api, modelzoo
    return api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build(model, 1)))


def _same(fmt, want):
    assert fmt["src_channel"] == want["src_channel"]
    np.testing.assert_array_equal(np.float32(fmt["mean"]), np.float32(want["mean"]))
    np.testing.assert_array_equal(np.float32(fmt["scale"]), np.float32(want["scale"]))


def test_image_format_survives_save_load_and_reset_batch_size():
    from anakin_b200 import api
    G = _graph()
    assert G.input_image("input_0") is None
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    _same(G.input_image("input_0"), FMT)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        G2 = api.Graph.from_file(p)
    _same(G2.input_image("input_0"), FMT)
    G2.ResetBatchSize("input_0", 8)
    G2.Reshape("input_0", [8, 3, 40, 48])
    G2.Optimize()
    _same(G2.input_image("input_0"), FMT)
    # identity channel order by default
    G.set_input_image("input_0", [1, 2, 3], [0.5, 0.25, 2.0])
    assert G.input_image("input_0")["src_channel"] == [0, 1, 2]


def test_set_input_image_rejects_bad_targets_and_formats():
    from anakin_b200 import anakin_bin, api, modelzoo
    G = _graph()
    with pytest.raises(api.AnakinError, match="not an Input"):
        G.set_input_image("conv1", [0, 0, 0], [1, 1, 1])
    with pytest.raises(api.AnakinError, match="no node"):
        G.set_input_image("no_such_input", [0, 0, 0], [1, 1, 1])
    with pytest.raises(api.AnakinError):
        G.set_input_image("input_0", [0, 0, 0], [1, 1, 1], [0, 0, 1])          # not a permutation
    with pytest.raises(api.AnakinError):
        G.set_input_image("input_0", [0, float("nan"), 0], [1, 1, 1])         # NaN mean
    with pytest.raises(api.AnakinError):
        G.set_input_image("input_0", [0, 0, 0], [1, float("inf"), 1])         # infinite scale
    with pytest.raises(api.AnakinError):
        G.set_input_image("input_0", [0, 0], [1, 1])                          # two entries for three channels
    with pytest.raises(api.AnakinError, match="one entry per channel"):
        G.set_input_image("input_0", [0] * 4, [1] * 4, [2, 1, 0, 3])          # four entries for three channels
    assert G.input_image("input_0") is None, "a rejected format must leave the input as it was"
    assert G.input_shape("input_0") == [1, 3, 32, 32]
    # a five-channel Input cannot be an image input
    b = modelzoo.GraphBuilder("five")
    x = b.input("input_0", (1, 5, 8, 8))
    x = b.conv("conv1", x, 5, 16, 3, 1, 1)
    b.output("out", x)
    G5 = api.Graph.from_bytes(anakin_bin.dumps(b.finalize()))
    with pytest.raises(api.AnakinError):
        G5.set_input_image("input_0", [0] * 4, [1] * 4)
    with pytest.raises(api.AnakinError):
        G5.set_input_image("input_0", [0] * 5, [1] * 5)


def _bad_descs(A):
    """Malformed formats only: each is rejected before the device check, so nothing is ever launched (a valid one
    would launch on a GPU machine, and these buffers are host memory)."""
    good = A.image_desc([1.0, 2.0, 3.0], [0.5, 0.5, 0.5], [2, 1, 0])
    d = A.image_desc([1.0, 2.0, 3.0], [0.5, 0.5, 0.5], [0, 0, 1])
    yield "not a permutation", d, 3
    d = A.image_desc([1.0, float("nan"), 3.0], [0.5, 0.5, 0.5])
    yield "NaN mean", d, 3
    d = A.image_desc([1.0, 2.0, 3.0], [0.5, float("-inf"), 0.5])
    yield "infinite scale", d, 3
    d = A.image_desc([1.0, 2.0, 3.0], [0.5, 0.5, 0.5], [0, 1, 3])
    yield "channel out of range", d, 3
    yield "c = 5", good, 5
    yield "c = 0", good, 0


def test_kernel_entry_points_validate_without_a_gpu():
    from anakin_b200 import saber_abi as A
    lib = A.load()
    buf = (C.c_uint8 * 4096)()
    p = C.cast(buf, C.c_void_p)
    for what, d, c in _bad_descs(A):
        want = A.INVALID_VALUE
        got = lib.b200_image_to_nhwc(C.byref(d), p, p, A.UINT8, 1, c, 4, 4, 16, 1.0, None)
        assert got == want, ("image_to_nhwc", what, got)
        sd = A.StemDesc()
        sd.math, sd.out_dtype = A.MATH_I8, A.UINT8
        sd.n, sd.c, sd.h, sd.w, sd.k, sd.ldc = 1, c, 16, 16, 16, 16
        sd.r = sd.s = 3
        sd.stride_h = sd.stride_w = 1
        got = lib.b200_stem_conv_run_image(C.byref(sd), C.byref(d), p, p, None, None, p, None)
        assert got == want, ("stem_conv_run_image", what, got)
    good = A.image_desc([1.0, 2.0, 3.0], [0.5, 0.5, 0.5])
    assert lib.b200_image_to_nhwc(None, p, p, A.UINT8, 1, 3, 4, 4, 16, 1.0, None) == A.INVALID_VALUE
    assert lib.b200_image_to_nhwc(C.byref(good), None, p, A.UINT8, 1, 3, 4, 4, 16, 1.0, None) == A.INVALID_VALUE
    assert lib.b200_image_to_nhwc(C.byref(good), p, None, A.UINT8, 1, 3, 4, 4, 16, 1.0, None) == A.INVALID_VALUE
    assert lib.b200_image_to_nhwc(C.byref(good), p, p, A.UINT8, 1, 3, 4, 4, 2, 1.0, None) == A.INVALID_VALUE
    sd = A.StemDesc()
    sd.c = 3
    assert lib.b200_stem_conv_run_image(None, C.byref(good), p, p, None, None, p, None) == A.INVALID_VALUE
    assert lib.b200_stem_conv_run_image(C.byref(sd), None, p, p, None, None, p, None) == A.INVALID_VALUE
    assert lib.b200_stem_conv_run_image(C.byref(sd), C.byref(good), None, p, None, None, p, None) == A.INVALID_VALUE
    assert lib.b200_stem_conv_run_image(C.byref(sd), C.byref(good), p, None, None, None, p, None) == A.INVALID_VALUE
    assert lib.b200_stem_conv_run_image(C.byref(sd), C.byref(good), p, p, None, None, None, None) == A.INVALID_VALUE
