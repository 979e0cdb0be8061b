"""CPU: NV12 / I420 sources of the on-device resize. The numpy restatement (tests/yuv_oracle.py) against the digests of
tests/golden/yuv_resize.json and, where cv2 imports, against OpenCV on every (Y, U, V) triple; the argument checks of
b200_image_resize_yuv_run / b200_image_resize_pil_yuv_run without a GPU; the image_pixel_format attribute."""
import ctypes as C
import hashlib
import json
import os
import tempfile

import numpy as np
import pytest

import pil_resize_oracle as P
import yuv_oracle as Y

HERE = os.path.dirname(os.path.abspath(__file__))
FMT = {"mean": [123.675, 116.28, 103.53], "scale": [1 / 58.395, 1 / 57.12, 1 / 57.375], "src_channel": [0, 1, 2]}


def _golden():
    with open(os.path.join(HERE, "golden", "yuv_resize.json")) as f:
        return json.load(f)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _case_id(c):
    return "%s_%dx%d_s%d_%dx%d" % (c["format"], c["h"], c["w"], c["resize_short"], c["out_h"], c["out_w"])


@pytest.mark.parametrize("name", sorted(Y.FORMATS))
def test_conversion_equals_fixture_on_every_triple(name):
    fmt = Y.FORMATS[name]
    frame = Y.exhaustive_frame(fmt)
    y, u, v = Y.planes(frame, fmt)
    up = lambda c: np.repeat(np.repeat(c, 2, axis=0), 2, axis=1).astype(np.int64)     # noqa: E731
    assert len(np.unique((y.astype(np.int64) << 16) | (up(u) << 8) | up(v))) == 1 << 24
    assert _sha(Y.yuv_to_rgb(frame, fmt)) == _golden()["exhaustive"][name]


@pytest.mark.parametrize("name", sorted(Y.FORMATS))
def test_conversion_equals_cv2_on_every_triple(name):
    pytest.importorskip("cv2")
    fmt = Y.FORMATS[name]
    frame = Y.exhaustive_frame(fmt)
    assert np.array_equal(Y.yuv_to_rgb(frame, fmt), Y.cv2_rgb(frame, fmt))


@pytest.mark.parametrize("case", _golden()["cases"], ids=_case_id)
def test_composed_restatement_equals_fixture(case):
    fmt = Y.FORMATS[case["format"]]
    frame = Y.golden_frame(case["h"], case["w"], fmt, case["index"])
    assert frame.shape == (case["h"] * 3 // 2, case["w"])
    got = Y.resize(frame, fmt, "pil", case["resize_short"], case["out_h"], case["out_w"])
    assert got.shape == (case["out_h"], case["out_w"], 3)
    assert _sha(got) == case["sha256"]


def test_fixture_covers_both_pass_orders_and_a_half_even_crop():
    hw = {(c["h"], c["w"], c["resize_short"]) for c in _golden()["cases"]}
    assert P.vertical_first(2000, 16, 224) and (2000, 16, 0) in hw
    assert not P.vertical_first(1600, 16, 224) and (1600, 16, 0) in hw
    rh, rw, _, left = P.geometry(480, 640, 256, 224, 224)
    assert (rw - 224) % 2 == 1 and left == round((rw - 224) / 2) and (480, 640, 256) in hw


def test_layouts_place_the_same_planes():
    """NV12 interleaves U,V after the Y plane; I420 puts the whole U plane, then V: the same planes, other bytes."""
    rng = np.random.default_rng(3)
    y = rng.integers(0, 256, (6, 8), dtype=np.uint8)
    u = rng.integers(0, 256, (3, 4), dtype=np.uint8)
    v = rng.integers(0, 256, (3, 4), dtype=np.uint8)
    nv12, i420 = Y.make_frame(y, u, v, Y.NV12), Y.make_frame(y, u, v, Y.I420)
    assert nv12.shape == i420.shape == (9, 8) and not np.array_equal(nv12, i420)
    assert np.array_equal(nv12[6:].reshape(3, 4, 2)[..., 1], v) and np.array_equal(i420[6:].reshape(-1)[12:], v.ravel())
    assert np.array_equal(Y.yuv_to_rgb(nv12, Y.NV12), Y.yuv_to_rgb(i420, Y.I420))


def _desc(A, n=2, c=3, oh=224, ow=224):
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = n, c, oh, ow
    return d


def test_run_entry_points_validate_arguments_without_a_gpu():
    from anakin_b200 import saber_abi as A
    lib = A.load()
    p = C.c_void_p(16)      # never dereferenced: argument errors are reported before any device work
    good = _desc(A)
    bad_descs = [_desc(A, c=1), _desc(A, c=4), _desc(A, n=0), _desc(A, oh=0), _desc(A, ow=0)]
    for fmt in (0, 3, -1):
        assert lib.b200_image_resize_yuv_run(C.byref(good), fmt, p, p, p, None) == A.INVALID_VALUE, fmt
        assert lib.b200_image_resize_pil_yuv_run(C.byref(good), fmt, 500, 500, 256, p, p, p, p,
                                                 None) == A.INVALID_VALUE, fmt
    for fmt in (A.IMAGE_YUV_NV12, A.IMAGE_YUV_I420):
        assert lib.b200_image_resize_yuv_run(None, fmt, p, p, p, None) == A.INVALID_VALUE
        for d in bad_descs:
            assert lib.b200_image_resize_yuv_run(C.byref(d), fmt, p, p, p, None) == A.INVALID_VALUE
            assert lib.b200_image_resize_pil_yuv_run(C.byref(d), fmt, 500, 500, 256, p, p, p, p,
                                                     None) == A.INVALID_VALUE
        for i in range(3):
            a = [p, p, p]
            a[i] = None
            assert lib.b200_image_resize_yuv_run(C.byref(good), fmt, *a, None) == A.INVALID_VALUE, i
        for i in range(4):
            a = [p, p, p, p]
            a[i] = None
            assert lib.b200_image_resize_pil_yuv_run(C.byref(good), fmt, 500, 500, 256, *a, None) == A.INVALID_VALUE
        for mh, mw, s in ((0, 500, 256), (500, 500, -1), (500, 500, 100)):
            assert lib.b200_image_resize_pil_yuv_run(C.byref(good), fmt, mh, mw, s, p, p, p, p,
                                                     None) == A.INVALID_VALUE


def test_pack_images_takes_cv2_layout_frames():
    from anakin_b200 import api
    frames = [Y.random_frame(4, 6, Y.NV12, 0), Y.random_frame(8, 2, Y.I420, 1)]
    pix, hw = api.pack_images(frames)
    assert hw.tolist() == [[4, 6], [8, 2]] and pix.size == 4 * 6 * 3 // 2 + 8 * 2 * 3 // 2
    assert np.array_equal(pix, np.concatenate([f.ravel() for f in frames]))
    with pytest.raises(api.AnakinError, match="YUV frames"):
        api.pack_images([np.zeros((5, 6), np.uint8)])          # not h * 3 / 2 rows


def _graph(c=3):
    from anakin_b200 import anakin_bin, api, modelzoo
    g = modelzoo.build("tiny_resnet", 1)
    G = api.Graph.from_bytes(anakin_bin.dumps(g))
    if c != 3:
        G.Reshape("input_0", [1, c] + G.input_shape("input_0")[2:])
    G.set_input_image("input_0", FMT["mean"][:c], FMT["scale"][:c], list(range(c)))
    return G


def test_pixel_format_survives_save_load_reshape_and_reset_batch_size():
    from anakin_b200 import api
    G = _graph()
    assert G.input_image_pixel_format("input_0") is None
    G.set_input_image_resize("input_0", 1080, 1920, 256, filter="pil", pixel_format="nv12")
    assert G.input_image_pixel_format("input_0") == "nv12"
    assert G.input_image_resize_filter("input_0") == "pil"
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        G2 = api.Graph.from_file(p)
    assert G2.input_image_pixel_format("input_0") == "nv12"
    G2.ResetBatchSize("input_0", 8)
    G2.Reshape("input_0", [8, 3, 40, 48])
    G2.Optimize()
    assert G2.input_image_pixel_format("input_0") == "nv12"
    assert G2.input_image_resize("input_0") == {"max_h": 1080, "max_w": 1920, "resize_short": 256}
    G2.set_input_image_resize("input_0", 720, 1280, 0, pixel_format="i420")
    assert G2.input_image_pixel_format("input_0") == "i420"
    G2.set_input_image_resize("input_0", 720, 1280, 0)
    assert G2.input_image_pixel_format("input_0") == "interleaved"


def test_pixel_format_absent_reads_as_interleaved_and_a_bad_stored_value_is_malformed():
    from anakin_b200 import anakin_bin, api
    G = _graph()
    G.set_input_image_resize("input_0", 96, 96, 36, pixel_format="i420")
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        with open(p, "rb") as f:
            g = anakin_bin.loads(f.read())
    node = next(n for n in g["nodes"] if n["op"] == "Input")
    assert node["attrs"]["image_pixel_format"] == 2
    del node["attrs"]["image_pixel_format"]
    assert api.Graph.from_bytes(anakin_bin.dumps(g)).input_image_pixel_format("input_0") == "interleaved"
    for bad in (3, -1):
        node["attrs"]["image_pixel_format"] = bad
        Gb = api.Graph.from_bytes(anakin_bin.dumps(g))
        assert Gb.input_image_pixel_format("input_0") is None
        assert Gb.input_image_resize("input_0") is None


def test_pixel_format_rejections():
    from anakin_b200 import api
    lib = api.load()
    G = _graph()
    for bad in ("yuv420p", "NV12", 1, None):
        with pytest.raises(api.AnakinError, match="pixel_format"):
            G.set_input_image_resize("input_0", 500, 500, 256, pixel_format=bad)
    assert G.input_image_resize("input_0") is None, "a rejected format must leave the input as it was"
    h = G._h
    assert lib.anakin_graph_set_input_image_pixel_format(h, b"input_0", 1) != 0       # resize attributes first
    assert b"set_input_image_resize first" in lib.anakin_last_error()
    assert lib.anakin_graph_input_image_pixel_format(h, b"input_0") == -1
    assert lib.anakin_graph_set_input_image_resize(h, b"input_0", 640, 480, 0) == 0
    assert lib.anakin_graph_input_image_pixel_format(h, b"input_0") == 0
    for bad in (3, -1, 1 << 30):
        assert lib.anakin_graph_set_input_image_pixel_format(h, b"input_0", bad) != 0
        assert b"format must be 0 (interleaved), 1 (nv12) or 2 (i420)" in lib.anakin_last_error()
    assert lib.anakin_graph_input_image_pixel_format(h, b"input_0") == 0
    for name in (b"conv1", b"nope"):
        assert lib.anakin_graph_set_input_image_pixel_format(h, name, 1) != 0
        assert lib.anakin_graph_input_image_pixel_format(h, name) == -1
    assert lib.anakin_graph_set_input_image_pixel_format(h, None, 1) != 0
    assert lib.anakin_graph_set_input_image_pixel_format(None, b"input_0", 1) != 0
    assert lib.anakin_graph_input_image_pixel_format(None, b"input_0") == -1
    assert lib.anakin_graph_set_input_image_pixel_format(h, b"input_0", 2) == 0
    assert lib.anakin_graph_input_image_pixel_format(h, b"input_0") == 2
    # the channel count is Net::init's to check: a 1-channel input takes the attribute
    G1 = _graph(c=1)
    G1.set_input_image_resize("input_0", 96, 96, 36, pixel_format="nv12")
    assert G1.input_image_pixel_format("input_0") == "nv12"
