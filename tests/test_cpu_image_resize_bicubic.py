"""CPU: Pillow's BICUBIC filter of the on-device resize (B200_IMAGE_RESIZE_PIL_BICUBIC, filter="pil_bicubic"). The
numpy restatement (tests/pil_bicubic_oracle.py) against the digests of
tests/golden/pil_bicubic_resize.json and against Pillow and torchvision; b200_image_resize_geometry_ex and the
workspace query b200_image_resize_workspace against the restatement; argument errors of the crop entry point; the
image_resize_filter attribute with value 3 through the C API and Python."""
import ctypes as C
import hashlib
import json
import os
import tempfile

import numpy as np
import pytest

import pil_bicubic_oracle as B
import pil_resize_oracle as P

HERE = os.path.dirname(os.path.abspath(__file__))
FMT = {"mean": [123.675, 116.28, 103.53], "scale": [1 / 58.395, 1 / 57.12, 1 / 57.375], "src_channel": [2, 1, 0]}
BICUBIC = 3


def _golden():
    with open(os.path.join(HERE, "golden", "pil_bicubic_resize.json")) as f:
        doc = json.load(f)
    assert doc["filter"] == "bicubic"
    return doc["cases"]


def _case_id(c):
    return "%dx%dx%d_s%d_%dx%d_%s" % (c["h"], c["w"], c["c"], c["resize_short"], c["out_h"], c["out_w"], c["image"])


def test_fixture_holds_the_designed_cases():
    want = [tuple(c) for c in B.GOLDEN_CASES]
    assert B.GOLDEN_CASES[:len(P.GOLDEN_CASES)] == list(P.GOLDEN_CASES)       # the bilinear fixture's cases first
    got = [(c["h"], c["w"], c["c"], c["resize_short"], c["out_h"], c["out_w"], c["image"]) for c in _golden()]
    assert got == want and [c["seed"] for c in _golden()] == list(range(len(want)))


@pytest.mark.parametrize("case", _golden(), ids=_case_id)
def test_restatement_equals_fixture(case):
    img = B.case_image(case["h"], case["w"], case["c"], case["image"], case["seed"])
    got = B.resize_u8(img, case["resize_short"], case["out_h"], case["out_w"])
    assert got.shape == (case["out_h"], case["out_w"], case["c"])
    assert hashlib.sha256(got.tobytes()).hexdigest() == case["sha256"]


@pytest.mark.parametrize("case", _golden(), ids=_case_id)
def test_restatement_equals_pillow(case):
    pytest.importorskip("PIL")
    pytest.importorskip("torchvision")
    img = B.case_image(case["h"], case["w"], case["c"], case["image"], case["seed"])
    want = B.pillow_resize(img, case["resize_short"], case["out_h"], case["out_w"])
    assert np.array_equal(B.resize_u8(img, case["resize_short"], case["out_h"], case["out_w"]), want)


def test_bicubic_differs_from_bilinear_only_in_the_filter():
    """Same geometry and pass order as the bilinear restatement; different taps and bytes."""
    img = P.case_image(375, 500, 3, "random", 0)
    assert not np.array_equal(P.resize_u8(img, 256, 224, 224), B.resize_u8(img, 256, 224, 224))
    xb, kb = B.coeffs(500, 341, [10, 11])
    xl, kl = P.coeffs(500, 341, [10, 11])
    assert kb.shape[1] == 2 * 3 + 1 and kl.shape[1] == 2 * 2 + 1      # support 2 * 1.47 against 1.47
    assert (xb < xl).all() and (np.abs(kb.sum(axis=1) - (1 << 22)) <= kb.shape[1]).all()


def test_cubic_filter_values():
    """Pillow's bicubic_filter (a = -0.5) at its knots and a few exact points."""
    for x, want in ((0.0, 1.0), (1.0, 0.0), (2.0, 0.0), (2.5, 0.0), (0.5, 0.5625), (1.5, -0.0625), (-1.5, -0.0625)):
        assert B.cubic(x) == want, x


def test_overshoot_leaves_the_byte_range_in_both_passes():
    """The checkerboard case: negative lobes push both passes' sums below 0 and above 255 * 2^22, where the clamp
    decides the byte, and the bytes are still Pillow's (test_restatement_equals_fixture)."""
    h, w, c, s, oh, ow, image = B.OVERSHOOT_CASE
    img = B.case_image(h, w, c, image, B.GOLDEN_CASES.index(B.OVERSHOOT_CASE))
    sums = []
    out = B.resize_u8(img, s, oh, ow, sums=sums)
    assert len(sums) == 2
    for acc in sums:
        assert acc.min() < 0 and acc.max() > 255 << B.PRECISION_BITS, (acc.min(), acc.max())
        assert np.abs(acc).max() < 2 ** 31
    assert out.min() == 0 and out.max() == 255
    k = B.coeffs(w, ow, np.arange(ow))[1]
    assert (k < 0).any()


def test_longest_tap_records():
    """1 x 16384 stretched to 224 x 224: 292 non-zero taps per column, against the workspace's kmax of 295 at the
    Net's 16384-pixel limit (149 for the bilinear filter)."""
    h, w, c, s, oh, ow, _ = B.LONGEST_CASE
    rh, rw, top, left = P.geometry(h, w, s, oh, ow)
    k = B.coeffs(w, rw, np.arange(ow) + left)[1]
    assert int((k != 0).sum(axis=1).max()) == 292
    assert k.shape[1] == B.kmax(16384, 224) == 295
    assert B.kmax(16384, 224, support=1) == 149


def _lib():
    from anakin_b200 import saber_abi as A
    return A, A.load()


def _geometry_ex(lib, h, w, s, oh, ow, filt):
    v = [C.c_int32(-7) for _ in range(4)]
    st = lib.b200_image_resize_geometry_ex(h, w, s, oh, ow, filt, *[C.byref(x) for x in v])
    return st, tuple(x.value for x in v)


def test_geometry_ex_equals_the_bilinear_geometry():
    A, lib = _lib()
    assert A.IMAGE_RESIZE_PIL_BICUBIC == BICUBIC
    rng = np.random.default_rng(11)
    cases = [(int(h), int(w)) for h, w in rng.integers(1, 5000, (200, 2))]
    cases += [(375, 500), (500, 375), (1, 1), (1, 16384), (16, 2000), (2000, 16), (4032, 3024), (1 << 23, 1)]
    for h, w in cases:
        for s, oh, ow in ((256, 224, 224), (232, 224, 224), (256, 200, 160), (0, 224, 224), (300, 225, 223),
                          (200, 224, 224)):
            st1, got1 = _geometry_ex(lib, h, w, s, oh, ow, A.IMAGE_RESIZE_PIL)
            st3, got3 = _geometry_ex(lib, h, w, s, oh, ow, BICUBIC)
            assert st3 == st1 and (st1 != A.SUCCESS or got3 == got1), (h, w, s, oh, ow)
            want = P.geometry(h, w, s, oh, ow)
            assert (st3 == A.SUCCESS) == (want is not None)
            if want is not None:
                assert got3 == want
    assert lib.b200_image_resize_geometry_ex(375, 500, 256, 224, 224, BICUBIC, None, None, None, None) == \
        A.INVALID_VALUE
    for filt in (-1, 2, 4):
        assert _geometry_ex(lib, 375, 500, 256, 224, 224, filt)[0] == A.INVALID_VALUE


def _desc(A, n=2, c=3, oh=224, ow=224):
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = n, c, oh, ow
    return d


def _workspace(lib, d, filt, max_h, max_w, s):
    b = C.c_size_t(12345)
    st = lib.b200_image_resize_workspace(C.byref(d) if d is not None else None, filt, max_h, max_w, s, C.byref(b))
    return st, b.value


def _want_workspace(n, c, oh, ow, max_h, max_w, s, filter):
    """The layout b200_image_resize_workspace documents for a Pillow filter: records of 2 + kmax int32 for every
    cropped row and column, then one intermediate per image (max_h rows of out_w or out_h rows of max_w pixels,
    padded to 4)."""
    up = lambda x, m: -(-x // m) * m        # noqa: E731
    mrh, mrw = (s, s) if s else (oh, ow)
    f = {"bilinear": 1, "bicubic": 2}[filter]
    kmax = max(B.kmax(max_h, mrh, f), B.kmax(max_w, mrw, f))
    coef = up(n * (oh + ow) * (2 + kmax) * 4, 256)
    tmp = up(max(max_h * up(ow, 4), oh * up(max_w, 4)) * c, 256)
    return coef + n * tmp, kmax


WORKSPACE_CASES = [(8, 3, 224, 224, 4032, 4032, 256), (32, 3, 224, 224, 1280, 1280, 256), (1, 1, 224, 221, 16384, 16384, 0),
                   (2, 4, 200, 160, 96, 3000, 232), (3, 2, 7, 5, 1, 1, 0), (1, 3, 224, 224, 1, 16384, 0),
                   (8, 3, 224, 224, 500, 500, 256), (4, 3, 224, 224, 224, 224, 224)]


def test_workspace_query_matches_the_layout():
    A, lib = _lib()
    for n, c, oh, ow, mh, mw, s in WORKSPACE_CASES:
        d = _desc(A, n, c, oh, ow)
        for filt, name in ((A.IMAGE_RESIZE_PIL, "bilinear"), (BICUBIC, "bicubic")):
            st, got = _workspace(lib, d, filt, mh, mw, s)
            assert st == A.SUCCESS and got == _want_workspace(n, c, oh, ow, mh, mw, s, name)[0], (filt, mh, mw, s)
        # the bilinear query is the old entry point's, unchanged
        old = C.c_size_t(0)
        assert lib.b200_image_resize_pil_workspace(C.byref(d), mh, mw, s, C.byref(old)) == A.SUCCESS
        assert old.value == _workspace(lib, d, A.IMAGE_RESIZE_PIL, mh, mw, s)[1]
        # the reference filter needs none, whatever the sizes
        assert _workspace(lib, d, A.IMAGE_RESIZE_REFERENCE, mh, mw, s) == (A.SUCCESS, 0)
        assert _workspace(lib, d, A.IMAGE_RESIZE_REFERENCE, 0, 0, -1) == (A.SUCCESS, 0)
    assert _want_workspace(1, 3, 224, 224, 16384, 16384, 0, "bicubic")[1] == 295
    assert _want_workspace(1, 3, 224, 224, 16384, 16384, 0, "bilinear")[1] == 149
    # an upscale still holds the cubic's 2 * 2 + 1 taps
    assert _want_workspace(1, 3, 224, 224, 7, 7, 0, "bicubic")[1] == 5


def test_every_restated_tap_count_fits_kmax():
    for h, w, s in ((4032, 3024, 256), (16384, 16384, 0), (16384, 1, 0), (1, 16384, 0), (1, 16384, 224),
                    (100, 150, 0), (7, 5, 0), (500, 375, 256), (257, 999, 256)):
        kmax = _want_workspace(1, 3, 224, 224, h, w, s, "bicubic")[1]
        rh, rw, top, left = P.geometry(h, w, s, 224, 224)
        for size, r, o in ((h, rh, top), (w, rw, left)):
            k = B.coeffs(size, r, np.arange(o, o + 224))[1]
            assert k.shape[1] <= kmax, (h, w, s, k.shape, kmax)


def test_workspace_query_rejections():
    A, lib = _lib()
    good = _desc(A)
    for filt in (-1, 2, 4, 99):
        assert _workspace(lib, good, filt, 500, 500, 256)[0] == A.INVALID_VALUE, filt
    for filt in (A.IMAGE_RESIZE_REFERENCE, A.IMAGE_RESIZE_PIL, BICUBIC):
        for d in (_desc(A, n=0), _desc(A, c=0), _desc(A, c=5), _desc(A, oh=0), _desc(A, ow=0)):
            assert _workspace(lib, d, filt, 500, 500, 256)[0] == A.INVALID_VALUE, filt
        assert _workspace(lib, None, filt, 500, 500, 256)[0] == A.INVALID_VALUE
        assert lib.b200_image_resize_workspace(C.byref(good), filt, 500, 500, 256, None) == A.INVALID_VALUE
    for filt in (A.IMAGE_RESIZE_PIL, BICUBIC):
        for mh, mw, s in ((0, 500, 256), (500, 0, 256), ((1 << 23) + 1, 500, 256), (500, 500, -1), (500, 500, 223)):
            assert _workspace(lib, good, filt, mh, mw, s)[0] == A.INVALID_VALUE, (filt, mh, mw, s)


def test_crop_run_validates_bicubic_arguments_without_a_gpu():
    A, lib = _lib()
    run = lib.b200_image_crop_resize_run
    p = C.c_void_p(16)      # never dereferenced: argument errors are reported before any device work
    good = _desc(A)
    for fmt in (A.IMAGE_INTERLEAVED, A.IMAGE_YUV_NV12, A.IMAGE_YUV_I420):
        assert run(None, BICUBIC, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
        for i in range(4):      # src, table, workspace, out
            a = [p, p, p, p]
            a[i] = None
            assert run(C.byref(good), BICUBIC, fmt, 500, 500, 256, *a, None) == A.INVALID_VALUE, (fmt, i)
        for d in (_desc(A, n=0), _desc(A, oh=0), _desc(A, ow=0), _desc(A, c=5)):
            assert run(C.byref(d), BICUBIC, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
        for mh, mw, s in ((0, 500, 256), (500, 0, 256), ((1 << 23) + 1, 500, 256), (500, 500, -1), (500, 500, 100)):
            assert run(C.byref(good), BICUBIC, fmt, mh, mw, s, p, p, p, p, None) == A.INVALID_VALUE, (fmt, mh, mw, s)
    for fmt in (-1, 3):
        assert run(C.byref(good), BICUBIC, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
    for fmt in (A.IMAGE_YUV_NV12, A.IMAGE_YUV_I420):
        for c in (1, 2, 4):
            assert run(C.byref(_desc(A, c=c)), BICUBIC, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE


def test_bilinear_only_entry_points_stay_bilinear():
    """b200_image_resize_pil_run and _pil_yuv_run take no filter; the bicubic filter runs through the crop entry
    point alone, and filter 2 stays unknown everywhere."""
    A, lib = _lib()
    p = C.c_void_p(16)
    assert lib.b200_image_crop_resize_run(C.byref(_desc(A)), 2, 0, 500, 500, 256, p, p, p, p, None) == \
        A.INVALID_VALUE
    assert _workspace(lib, _desc(A), 2, 500, 500, 256)[0] == A.INVALID_VALUE


def _graph():
    from anakin_b200 import anakin_bin, api, modelzoo
    return api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build("tiny_resnet", 1)))


def test_filter_attribute_survives_save_load_reshape_and_reset_batch_size():
    from anakin_b200 import anakin_bin, api
    assert api.RESIZE_FILTERS["pil_bicubic"] == BICUBIC
    G = _graph()
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    G.set_input_image_resize("input_0", 1280, 960, 256, filter="pil_bicubic")
    want = {"max_h": 1280, "max_w": 960, "resize_short": 256}
    assert G.input_image_resize("input_0") == want
    assert G.input_image_resize_filter("input_0") == "pil_bicubic"
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        G2 = api.Graph.from_file(p)
        with open(p, "rb") as f:
            g = anakin_bin.loads(f.read())
    node = next(n for n in g["nodes"] if n["op"] == "Input")
    assert node["attrs"]["image_resize_filter"] == BICUBIC
    assert G2.input_image_resize_filter("input_0") == "pil_bicubic"
    G2.ResetBatchSize("input_0", 8)
    G2.Reshape("input_0", [8, 3, 40, 48])
    G2.Optimize()
    assert G2.input_image_resize_filter("input_0") == "pil_bicubic"
    assert G2.input_image_resize("input_0") == want
    G2.set_input_image_resize("input_0", 640, 480, 0, filter="pil")
    assert G2.input_image_resize_filter("input_0") == "pil"
    G2.set_input_image_resize("input_0", 640, 480, 0, filter="pil_bicubic")
    assert G2.input_image_resize_filter("input_0") == "pil_bicubic"


def test_filter_c_api_accepts_and_reports_3():
    from anakin_b200 import api
    lib = api.load()
    G = _graph()
    h = G._h
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    assert lib.anakin_graph_set_input_image_resize_filter(h, b"input_0", BICUBIC) != 0    # resize attributes first
    assert b"set_input_image_resize first" in lib.anakin_last_error()
    assert lib.anakin_graph_set_input_image_resize(h, b"input_0", 640, 480, 0) == 0
    assert lib.anakin_graph_set_input_image_resize_filter(h, b"input_0", BICUBIC) == 0
    assert lib.anakin_graph_input_image_resize_filter(h, b"input_0") == BICUBIC
    for bad in (2, 4, -1):
        assert lib.anakin_graph_set_input_image_resize_filter(h, b"input_0", bad) != 0
        err = lib.anakin_last_error()
        assert b"filter must be 0 (reference) or 1 (pil)" in err and b"3 (pil_bicubic)" in err
        assert lib.anakin_graph_input_image_resize_filter(h, b"input_0") == BICUBIC      # unchanged
    for bad in ("bicubic", "PIL_BICUBIC", 3):
        with pytest.raises(api.AnakinError, match="filter"):
            G.set_input_image_resize("input_0", 500, 500, 256, filter=bad)
    assert G.input_image_resize_filter("input_0") == "pil_bicubic"
