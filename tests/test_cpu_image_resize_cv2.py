"""CPU: OpenCV's INTER_LINEAR filter of the on-device resize (B200_IMAGE_RESIZE_CV2_LINEAR, filter="cv2_linear"). The
numpy restatement (tests/cv2_resize_oracle.py) against the digests of tests/golden/cv2_resize.json and, where cv2
imports, against cv2.resize on seeded random sweeps; b200_image_resize_geometry_ex and the workspace query for the
filter; argument errors of the crop entry point; the image_resize_filter attribute with value 5 through the C API and
Python.

The filter refuses no case beyond the geometry's own limits (b200_image_resize_geometry): the sweeps below cover
upscales and shrinks of each axis, equal sizes and exact 2x shrinks, and every one equals cv2."""
import ctypes as C
import hashlib
import json
import os
import tempfile

import numpy as np
import pytest

import cv2_resize_oracle as O
import image_resize_oracle as R

HERE = os.path.dirname(os.path.abspath(__file__))
FMT = {"mean": [123.675, 116.28, 103.53], "scale": [1 / 58.395, 1 / 57.12, 1 / 57.375], "src_channel": [2, 1, 0]}
CV2_LINEAR = 5


def _golden():
    with open(os.path.join(HERE, "golden", "cv2_resize.json")) as f:
        doc = json.load(f)
    assert doc["filter"] == "cv2_linear"
    return doc["cases"]


def _case_id(c):
    return "%dx%dx%d_s%d_%dx%d_%s" % (c["h"], c["w"], c["c"], c["resize_short"], c["out_h"], c["out_w"], c["image"])


def test_fixture_holds_the_designed_cases():
    got = [(c["h"], c["w"], c["c"], c["resize_short"], c["out_h"], c["out_w"], c["image"]) for c in _golden()]
    assert got == [tuple(c) for c in O.GOLDEN_CASES]
    assert [c["seed"] for c in _golden()] == list(range(len(got)))


@pytest.mark.parametrize("case", _golden(), ids=_case_id)
def test_restatement_equals_fixture(case):
    src = O.case_image(case["h"], case["w"], case["c"], case["image"], case["seed"])
    got = O.case_resize(src, case["c"], case["image"], case["resize_short"], case["out_h"], case["out_w"])
    assert got.shape == (case["out_h"], case["out_w"], case["c"])
    assert hashlib.sha256(got.tobytes()).hexdigest() == case["sha256"]


@pytest.mark.parametrize("case", _golden(), ids=_case_id)
def test_restatement_equals_cv2(case):
    pytest.importorskip("cv2")
    src = O.case_image(case["h"], case["w"], case["c"], case["image"], case["seed"])
    args = (src, case["c"], case["image"], case["resize_short"], case["out_h"], case["out_w"])
    assert np.array_equal(O.case_resize(*args), O.case_resize(*args, cv2=True))


def _direction(a, b):
    return "up" if b > a else "down" if b < a else "equal"


def test_random_sweep_equals_cv2():
    """1,200 seeded stretches (whole resized images, no crop), c = 1..4, sides 1..120 each way: every mix of upscale,
    shrink and equal size over the two axes, and the exact 2x shrinks of every channel count."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2026)
    seen = {}
    cases = [(int(rng.integers(1, 5)),) + tuple(int(v) for v in rng.integers(1, 121, 4)) for _ in range(1150)]
    cases += [(c, 2 * h, 2 * w, h, w) for c in (1, 2, 3, 4) for h, w in ((1, 1), (3, 8), (16, 5), (37, 60))]
    cases += [(c, h, w, h, w2) for c in (1, 2, 3, 4) for h, w, w2 in ((20, 30, 30), (1, 9, 9), (40, 1, 2))]
    cases += [(c, h, w, h2, w) for c in (1, 2, 3, 4) for h, w, h2 in ((30, 20, 31), (9, 1, 3), (2, 40, 2))]
    for c, h, w, rh, rw in cases:
        img = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
        want = cv2.resize(img, (rw, rh), interpolation=cv2.INTER_LINEAR).reshape(rh, rw, c)
        got = O.resize_window(img, rh, rw, 0, 0, rh, rw)
        assert np.array_equal(got, want), (c, h, w, rh, rw)
        key = (_direction(h, rh), _direction(w, rw))
        seen[key] = seen.get(key, 0) + 1
    assert len(cases) >= 1000
    assert all(seen.get((a, b), 0) >= 3 for a in ("up", "down", "equal") for b in ("up", "down", "equal")), seen
    assert min(seen[k] for k in (("up", "up"), ("up", "down"), ("down", "up"), ("down", "down"))) >= 200


def test_random_short_side_crops_equal_cv2():
    """Short side + centre crop on larger images: the cropped window of cv2.resize at the floor offsets."""
    pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    for _ in range(60):
        c = int(rng.integers(1, 5))
        h, w = (int(v) for v in rng.integers(1, 1500, 2))
        s, oh, ow = [(256, 224, 224), (232, 224, 224), (300, 225, 223), (0, 224, 224), (0, 97, 301)][rng.integers(5)]
        img = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
        assert np.array_equal(O.resize_u8(img, s, oh, ow), O.cv2_resize(img, s, oh, ow)), (c, h, w, s, oh, ow)


def test_borders_of_an_upscale_weight_one_row_twice():
    """Rows keep the unclamped fraction: the first row of a 2 -> 5 upscale reads source row 0 twice with weights that
    sum to 2048, and the columns' first tap reads pixel 0 alone."""
    s0, s1, b0, b1 = O.axis(2, 5, [0], columns=False)
    assert (s0[0], s1[0]) == (0, 0) and b0[0] + b1[0] == 2048 and b1[0] > 0
    x0, x1, a0, a1 = O.axis(2, 5, [0], columns=True)
    assert (x0[0], a0[0], a1[0]) == (0, 2048, 0)
    x0, x1, a0, a1 = O.axis(2, 5, [4], columns=True)
    assert (x0[0], a0[0], a1[0]) == (1, 2048, 0)


def test_two_channel_2x_shrink_rounds_half_to_even():
    img = np.array([[[1, 2], [0, 0]], [[0, 0], [1, 4]]], np.uint8)       # block sums 2 (0.5) and 6 (1.5)
    assert O.resize_window(img, 1, 1, 0, 0, 1, 1).tolist() == [[[0, 2]]]
    assert O.resize_window(img[..., :1].repeat(3, axis=2), 1, 1, 0, 0, 1, 1).tolist() == [[[1, 1, 1]]]


def _lib():
    from anakin_b200 import saber_abi as A
    return A, A.load()


def _geometry_ex(lib, h, w, s, oh, ow, filt):
    v = [C.c_int32(-7) for _ in range(4)]
    st = lib.b200_image_resize_geometry_ex(h, w, s, oh, ow, filt, *[C.byref(x) for x in v])
    return st, tuple(x.value for x in v)


def test_geometry_ex_is_the_reference_geometry():
    A, lib = _lib()
    assert A.IMAGE_RESIZE_CV2_LINEAR == CV2_LINEAR
    rng = np.random.default_rng(12)
    cases = [(int(h), int(w)) for h, w in rng.integers(1, 5000, (200, 2))]
    cases += [(375, 500), (500, 375), (1, 1), (1, 16384), (4032, 3024), (1 << 23, 1), ((1 << 23) + 1, 1)]
    for h, w in cases:
        for s, oh, ow in ((256, 224, 224), (232, 224, 224), (300, 225, 223), (0, 224, 224), (200, 224, 224)):
            st, got = _geometry_ex(lib, h, w, s, oh, ow, CV2_LINEAR)
            st0, got0 = _geometry_ex(lib, h, w, s, oh, ow, A.IMAGE_RESIZE_REFERENCE)
            want = R.geometry(h, w, s, oh, ow)
            assert st == st0 and (st == A.SUCCESS) == (want is not None), (h, w, s, oh, ow)
            if want is not None:
                assert got == got0 == want
    # floor offsets, where Pillow's filters round half to even: 1920 x 1080 at S = 256 is 455 x 256, margin 231
    assert _geometry_ex(lib, 1080, 1920, 256, 224, 224, CV2_LINEAR)[1] == (256, 455, 16, 115)
    assert _geometry_ex(lib, 1080, 1920, 256, 224, 224, A.IMAGE_RESIZE_PIL)[1] == (256, 455, 16, 116)
    assert lib.b200_image_resize_geometry_ex(375, 500, 256, 224, 224, CV2_LINEAR, None, None, None, None) == \
        A.INVALID_VALUE
    for filt in (-1, 2, 4, 6):
        assert _geometry_ex(lib, 375, 500, 256, 224, 224, filt)[0] == A.INVALID_VALUE


def _desc(A, n=2, c=3, oh=224, ow=224):
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = n, c, oh, ow
    return d


def test_workspace_is_zero_bytes():
    A, lib = _lib()
    for n, c, oh, ow, mh, mw, s in ((8, 3, 224, 224, 4032, 4032, 256), (1, 1, 224, 221, 16384, 16384, 0),
                                    (3, 2, 7, 5, 1, 1, 0), (2, 4, 200, 160, 0, 0, -1)):
        b = C.c_size_t(12345)
        assert lib.b200_image_resize_workspace(C.byref(_desc(A, n, c, oh, ow)), CV2_LINEAR, mh, mw, s,
                                               C.byref(b)) == A.SUCCESS
        assert b.value == 0
    for d in (_desc(A, n=0), _desc(A, c=0), _desc(A, c=5), _desc(A, oh=0), _desc(A, ow=0)):
        assert lib.b200_image_resize_workspace(C.byref(d), CV2_LINEAR, 500, 500, 256, C.byref(b)) == A.INVALID_VALUE
    assert lib.b200_image_resize_workspace(None, CV2_LINEAR, 500, 500, 256, C.byref(b)) == A.INVALID_VALUE
    assert lib.b200_image_resize_workspace(C.byref(_desc(A)), CV2_LINEAR, 500, 500, 256, None) == A.INVALID_VALUE
    for filt in (4, 6):
        assert lib.b200_image_resize_workspace(C.byref(_desc(A)), filt, 500, 500, 256, C.byref(b)) == \
            A.INVALID_VALUE


def test_crop_run_validates_arguments_without_a_gpu():
    A, lib = _lib()
    run = lib.b200_image_crop_resize_run
    p = C.c_void_p(16)      # never dereferenced: argument errors are reported before any device work
    good = _desc(A)
    for fmt in (A.IMAGE_INTERLEAVED, A.IMAGE_YUV_NV12, A.IMAGE_YUV_I420):
        assert run(None, CV2_LINEAR, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
        for i in (0, 1, 3):      # src, table, out (the workspace is not read)
            a = [p, p, p, p]
            a[i] = None
            assert run(C.byref(good), CV2_LINEAR, fmt, 500, 500, 256, *a, None) == A.INVALID_VALUE, (fmt, i)
        for d in (_desc(A, n=0), _desc(A, oh=0), _desc(A, ow=0), _desc(A, c=5)):
            assert run(C.byref(d), CV2_LINEAR, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
    for fmt in (-1, 3):
        assert run(C.byref(good), CV2_LINEAR, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
    for fmt in (A.IMAGE_YUV_NV12, A.IMAGE_YUV_I420):
        for c in (1, 2, 4):
            assert run(C.byref(_desc(A, c=c)), CV2_LINEAR, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
    for filt in (4, 6):
        assert run(C.byref(good), filt, 0, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE


def _graph():
    from anakin_b200 import anakin_bin, api, modelzoo
    return api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build("tiny_resnet", 1)))


def test_filter_attribute_survives_save_load_reshape_and_reset_batch_size():
    from anakin_b200 import anakin_bin, api
    assert api.RESIZE_FILTERS["cv2_linear"] == CV2_LINEAR
    G = _graph()
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    G.set_input_image_resize("input_0", 1280, 960, 256, filter="cv2_linear", pixel_format="nv12")
    want = {"max_h": 1280, "max_w": 960, "resize_short": 256}
    assert G.input_image_resize("input_0") == want
    assert G.input_image_resize_filter("input_0") == "cv2_linear"
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        G2 = api.Graph.from_file(p)
        with open(p, "rb") as f:
            g = anakin_bin.loads(f.read())
    node = next(n for n in g["nodes"] if n["op"] == "Input")
    assert node["attrs"]["image_resize_filter"] == CV2_LINEAR
    assert G2.input_image_resize_filter("input_0") == "cv2_linear"
    assert G2.input_image_pixel_format("input_0") == "nv12"
    G2.ResetBatchSize("input_0", 8)
    G2.Reshape("input_0", [8, 3, 40, 48])
    G2.Optimize()
    assert G2.input_image_resize_filter("input_0") == "cv2_linear"
    assert G2.input_image_resize("input_0") == want
    G2.set_input_image_resize("input_0", 640, 480, 0, filter="pil")
    assert G2.input_image_resize_filter("input_0") == "pil"
    G2.set_input_image_resize("input_0", 640, 480, 0, filter="cv2_linear")
    assert G2.input_image_resize_filter("input_0") == "cv2_linear"


def test_filter_c_api_accepts_and_reports_5():
    from anakin_b200 import api
    lib = api.load()
    G = _graph()
    h = G._h
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    assert lib.anakin_graph_set_input_image_resize_filter(h, b"input_0", CV2_LINEAR) != 0    # resize attributes first
    assert lib.anakin_graph_set_input_image_resize(h, b"input_0", 640, 480, 0) == 0
    assert lib.anakin_graph_set_input_image_resize_filter(h, b"input_0", CV2_LINEAR) == 0
    assert lib.anakin_graph_input_image_resize_filter(h, b"input_0") == CV2_LINEAR
    for bad in (2, 4, 6, -1):
        assert lib.anakin_graph_set_input_image_resize_filter(h, b"input_0", bad) != 0
        assert b"5 (cv2_linear)" in lib.anakin_last_error()
        assert lib.anakin_graph_input_image_resize_filter(h, b"input_0") == CV2_LINEAR      # unchanged
    for bad in ("cv2", "INTER_LINEAR", "linear", 5):
        with pytest.raises(api.AnakinError, match="filter"):
            G.set_input_image_resize("input_0", 500, 500, 256, filter=bad)
    assert G.input_image_resize_filter("input_0") == "cv2_linear"
