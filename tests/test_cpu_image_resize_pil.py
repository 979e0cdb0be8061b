"""CPU: the Pillow filter of the on-device resize. The numpy restatement (tests/pil_resize_oracle.py) against Pillow
and torchvision and against the digests of tests/golden/pil_resize.json; b200_image_resize_geometry_ex and the
workspace query against the restatement; the image_resize_filter attribute; every rejection without a GPU."""
import ctypes as C
import hashlib
import json
import os
import tempfile

import numpy as np
import pytest

import image_resize_oracle as R
import pil_resize_oracle as P

HERE = os.path.dirname(os.path.abspath(__file__))
FMT = {"mean": [123.675, 116.28, 103.53], "scale": [1 / 58.395, 1 / 57.12, 1 / 57.375], "src_channel": [2, 1, 0]}


def _golden():
    with open(os.path.join(HERE, "golden", "pil_resize.json")) as f:
        return json.load(f)["cases"]


def _case_id(c):
    return "%dx%dx%d_s%d_%dx%d_%s" % (c["h"], c["w"], c["c"], c["resize_short"], c["out_h"], c["out_w"], c["image"])


@pytest.mark.parametrize("case", _golden(), ids=_case_id)
def test_restatement_equals_fixture(case):
    img = P.case_image(case["h"], case["w"], case["c"], case["image"], case["seed"])
    got = P.resize_u8(img, case["resize_short"], case["out_h"], case["out_w"])
    assert got.shape == (case["out_h"], case["out_w"], case["c"])
    assert hashlib.sha256(got.tobytes()).hexdigest() == case["sha256"]


@pytest.mark.parametrize("case", _golden(), ids=_case_id)
def test_restatement_equals_pillow(case):
    pytest.importorskip("PIL")
    pytest.importorskip("torchvision")
    img = P.case_image(case["h"], case["w"], case["c"], case["image"], case["seed"])
    want = P.pillow_resize(img, case["resize_short"], case["out_h"], case["out_w"])
    assert np.array_equal(P.resize_u8(img, case["resize_short"], case["out_h"], case["out_w"]), want)


@pytest.mark.parametrize("h,w,oh,ow", P.PASS_ORDER_CASES)
def test_pass_order_is_observable(h, w, oh, ow):
    """Each pass-order case tells the two orders apart, so the fixture pins the rule on both sides of the switch."""
    img = P.case_image(h, w, 3, "random", seed=h * w + oh)
    want_v = h > 100 * w and oh < h
    assert P.vertical_first(h, w, oh) == want_v
    assert not np.array_equal(P.resize_u8(img, 0, oh, ow, vfirst=True), P.resize_u8(img, 0, oh, ow, vfirst=False))


def test_antialiasing_on_a_phone_photo():
    """Fine stripes shrunk 12x average out under the Pillow filter; the reference filter aliases them."""
    img = P.case_image(3024, 4032, 3, "stripes", 0)
    pil = P.resize_u8(img, 256, 224, 224).astype(float)
    ref = R.image_resize_u8(img, 256, 224, 224).astype(float)
    assert pil.std() < 10 and ref.std() > 25, (pil.std(), ref.std())


def _lib():
    from anakin_b200 import saber_abi as A
    return A, A.load()


def _geometry_ex(lib, h, w, s, oh, ow, filt):
    v = [C.c_int32(-7) for _ in range(4)]
    st = lib.b200_image_resize_geometry_ex(h, w, s, oh, ow, filt, *[C.byref(x) for x in v])
    return st, tuple(x.value for x in v)


def test_geometry_ex_equals_restatement():
    A, lib = _lib()
    rng = np.random.default_rng(5)
    cases = [(int(h), int(w)) for h, w in rng.integers(1, 5000, (300, 2))]
    cases += [(375, 500), (500, 375), (1, 1), (16, 2000), (2000, 16), (4032, 3024), (1 << 23, 1), (1, 1 << 23)]
    for h, w in cases:
        for s, oh, ow in ((256, 224, 224), (232, 224, 224), (256, 200, 160), (0, 224, 224), (300, 225, 223)):
            st, got = _geometry_ex(lib, h, w, s, oh, ow, 1)
            want = P.geometry(h, w, s, oh, ow)
            assert (st == A.SUCCESS) == (want is not None), (h, w, s)
            if want is not None:
                assert got == want, (h, w, s, oh, ow, got, want)
            # filter 0 is b200_image_resize_geometry itself
            st0, got0 = _geometry_ex(lib, h, w, s, oh, ow, 0)
            assert (st0 == A.SUCCESS) == (want is not None)
            if want is not None:
                assert got0 == R.geometry(h, w, s, oh, ow)


@pytest.mark.parametrize("s,rw,want_left", [(256, 224 + 115, 58), (256, 224 + 117, 58), (256, 224 + 113, 56),
                                            (256, 224 + 119, 60), (256, 224 + 116, 58), (224, 224 + 1, 0),
                                            (224, 224 + 3, 2)])
def test_geometry_ex_crop_rounds_half_to_even(s, rw, want_left):
    """Odd rw - W puts the centre on a half, which rounds to even: 57.5 -> 58 and 58.5 -> 58, where the reference
    filter's floor gives 57 and 58."""
    A, lib = _lib()
    st, (rh, rw_, top, left) = _geometry_ex(lib, s, rw, s, 224, 224, 1)    # an s x rw image keeps its width
    assert st == A.SUCCESS and (rh, rw_, top) == (s, rw, (s - 224) // 2)
    assert left == want_left == round((rw - 224) / 2)
    assert _geometry_ex(lib, s, rw, s, 224, 224, 0)[1][3] == (rw - 224) // 2
    st, (rh, rw_, top, left) = _geometry_ex(lib, rw, s, s, 224, 224, 1)    # the same along the rows
    assert st == A.SUCCESS and rh == rw and top == want_left


def test_geometry_ex_rejections():
    A, lib = _lib()
    for filt in (-1, 2, 99):
        assert _geometry_ex(lib, 375, 500, 256, 224, 224, filt)[0] == A.INVALID_VALUE
    assert _geometry_ex(lib, 375, 500, 200, 224, 224, 1)[0] == A.INVALID_VALUE     # S below the crop
    assert _geometry_ex(lib, 0, 500, 256, 224, 224, 1)[0] == A.INVALID_VALUE
    assert lib.b200_image_resize_geometry_ex(375, 500, 256, 224, 224, 1, None, None, None, None) == A.INVALID_VALUE


def _desc(A, n=2, c=3, oh=224, ow=224):
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = n, c, oh, ow
    return d


def _workspace(A, lib, d, max_h, max_w, s):
    b = C.c_size_t(0)
    st = lib.b200_image_resize_pil_workspace(C.byref(d) if d is not None else None, max_h, max_w, s, C.byref(b))
    return st, b.value


def _want_workspace(n, c, oh, ow, max_h, max_w, s):
    """The layout b200_image_resize_pil_workspace documents: records of 2 + kmax int32 for every cropped row and
    column, then one intermediate per image (max_h rows of out_w or out_h rows of max_w pixels, padded to 4)."""
    up = lambda x, m: -(-x // m) * m        # noqa: E731
    mrh, mrw = (s, s) if s else (oh, ow)
    kmax = 2 * max(-(-max_h // mrh), -(-max_w // mrw), 1) + 1
    coef = up(n * (oh + ow) * (2 + kmax) * 4, 256)
    tmp = up(max(max_h * up(ow, 4), oh * up(max_w, 4)) * c, 256)
    return coef + n * tmp, kmax


def test_workspace_size():
    A, lib = _lib()
    for n, c, oh, ow, mh, mw, s in ((8, 3, 224, 224, 4032, 4032, 256), (32, 3, 224, 224, 1280, 1280, 256),
                                    (1, 1, 224, 221, 16384, 16384, 0), (2, 4, 200, 160, 96, 3000, 232),
                                    (3, 2, 7, 5, 1, 1, 0)):
        st, got = _workspace(A, lib, _desc(A, n, c, oh, ow), mh, mw, s)
        want, kmax = _want_workspace(n, c, oh, ow, mh, mw, s)
        assert st == A.SUCCESS and got == want, (n, c, oh, ow, mh, mw, s, got, want)
    # the largest tap count the records hold: 2 * ceil(16384 / 224) + 1 at the kMaxSide limit
    assert _want_workspace(1, 3, 224, 224, 16384, 16384, 0)[1] == 149
    # every tap count of the restatement fits kmax
    for h, w, s in ((4032, 3024, 256), (16384, 16384, 0), (16384, 1, 0), (1, 16384, 224), (100, 150, 0)):
        kmax = _want_workspace(1, 3, 224, 224, max(h, 1), max(w, 1), s)[1]
        rh, rw, top, left = P.geometry(h, w, s, 224, 224)
        assert P.coeffs(h, rh, [top, top + 223])[1].shape[1] <= kmax
        assert P.coeffs(w, rw, [left, left + 223])[1].shape[1] <= kmax


def test_workspace_and_run_validate_arguments_without_a_gpu():
    A, lib = _lib()
    bad_descs = [_desc(A, n=0), _desc(A, c=0), _desc(A, c=5), _desc(A, oh=0), _desc(A, ow=0)]
    for d in bad_descs:
        assert _workspace(A, lib, d, 500, 500, 256)[0] == A.INVALID_VALUE
    for mh, mw, s in ((0, 500, 256), (500, 0, 256), ((1 << 23) + 1, 500, 256), (500, 500, -1), (500, 500, 223)):
        assert _workspace(A, lib, _desc(A), mh, mw, s)[0] == A.INVALID_VALUE, (mh, mw, s)
    assert _workspace(A, lib, None, 500, 500, 256)[0] == A.INVALID_VALUE
    assert lib.b200_image_resize_pil_workspace(C.byref(_desc(A)), 500, 500, 256, None) == A.INVALID_VALUE
    p = C.c_void_p(16)      # never dereferenced: argument errors are reported before any device work
    good = _desc(A)
    args = [good, 500, 500, 256, p, p, p, p]
    for i in (0, 4, 5, 6, 7):
        a = list(args)
        a[i] = None
        assert lib.b200_image_resize_pil_run(*[C.byref(x) if isinstance(x, A.ImageResizeDesc) else x for x in a],
                                             None) == A.INVALID_VALUE, i
    for d in bad_descs:
        assert lib.b200_image_resize_pil_run(C.byref(d), 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
    for mh, mw, s in ((0, 500, 256), (500, 500, -1), (500, 500, 100)):
        assert lib.b200_image_resize_pil_run(C.byref(good), mh, mw, s, p, p, p, p, None) == A.INVALID_VALUE


def _graph():
    from anakin_b200 import anakin_bin, api, modelzoo
    return api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build("tiny_resnet", 1)))


def test_filter_attribute_survives_save_load_reshape_and_reset_batch_size():
    from anakin_b200 import api
    G = _graph()
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    assert G.input_image_resize_filter("input_0") is None
    G.set_input_image_resize("input_0", 1280, 960, 256)
    assert G.input_image_resize_filter("input_0") == "reference"
    G.set_input_image_resize("input_0", 1280, 960, 256, filter="pil")
    want = {"max_h": 1280, "max_w": 960, "resize_short": 256}
    assert G.input_image_resize("input_0") == want          # the getter keeps its return value
    assert G.input_image_resize_filter("input_0") == "pil"
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        G2 = api.Graph.from_file(p)
    assert G2.input_image_resize_filter("input_0") == "pil"
    G2.ResetBatchSize("input_0", 8)
    G2.Reshape("input_0", [8, 3, 40, 48])
    G2.Optimize()
    assert G2.input_image_resize_filter("input_0") == "pil"
    assert G2.input_image_resize("input_0") == want
    G2.set_input_image_resize("input_0", 640, 480, 0, filter="reference")
    assert G2.input_image_resize_filter("input_0") == "reference"


def test_filter_absent_reads_as_reference_and_a_bad_stored_value_is_malformed():
    from anakin_b200 import anakin_bin, api
    G = _graph()
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    G.set_input_image_resize("input_0", 96, 96, 36, filter="pil")
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        with open(p, "rb") as f:
            g = anakin_bin.loads(f.read())
    node = next(n for n in g["nodes"] if n["op"] == "Input")
    assert node["attrs"]["image_resize_filter"] == 1
    del node["attrs"]["image_resize_filter"]
    assert api.Graph.from_bytes(anakin_bin.dumps(g)).input_image_resize_filter("input_0") == "reference"
    for bad in (2, -1):
        node["attrs"]["image_resize_filter"] = bad
        Gb = api.Graph.from_bytes(anakin_bin.dumps(g))
        assert Gb.input_image_resize_filter("input_0") is None
        assert Gb.input_image_resize("input_0") is None


def test_filter_rejections_python():
    from anakin_b200 import api
    G = _graph()
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    for bad in ("bilinear", "PIL", 1, None):
        with pytest.raises(api.AnakinError, match="filter"):
            G.set_input_image_resize("input_0", 500, 500, 256, filter=bad)
    assert G.input_image_resize("input_0") is None, "a rejected filter must leave the input as it was"
    assert G.input_image_resize_filter("conv1") is None
    assert G.input_image_resize_filter("no_such_input") is None


def test_filter_rejections_c_api():
    from anakin_b200 import api
    lib = api.load()
    G = _graph()
    h = G._h
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    assert lib.anakin_graph_set_input_image_resize_filter(h, b"input_0", 1) != 0      # resize attributes first
    assert b"set_input_image_resize first" in lib.anakin_last_error()
    assert lib.anakin_graph_input_image_resize_filter(h, b"input_0") == -1
    assert lib.anakin_graph_set_input_image_resize(h, b"input_0", 640, 480, 0) == 0
    assert lib.anakin_graph_input_image_resize_filter(h, b"input_0") == 0
    for bad in (2, -1, 1 << 30):
        assert lib.anakin_graph_set_input_image_resize_filter(h, b"input_0", bad) != 0
        assert b"filter must be 0 (reference) or 1 (pil)" in lib.anakin_last_error()
    assert lib.anakin_graph_input_image_resize_filter(h, b"input_0") == 0
    for name in (b"conv1", b"nope"):
        assert lib.anakin_graph_set_input_image_resize_filter(h, name, 1) != 0
        assert lib.anakin_graph_input_image_resize_filter(h, name) == -1
    assert lib.anakin_graph_set_input_image_resize_filter(h, None, 1) != 0
    assert lib.anakin_graph_set_input_image_resize_filter(None, b"input_0", 1) != 0
    assert lib.anakin_graph_input_image_resize_filter(None, b"input_0") == -1
    assert lib.anakin_graph_set_input_image_resize_filter(h, b"input_0", 1) == 0
    assert lib.anakin_graph_input_image_resize_filter(h, b"input_0") == 1
    v = [C.c_int(-5) for _ in range(3)]
    assert lib.anakin_graph_input_image_resize(h, b"input_0", *[C.byref(x) for x in v]) == 1
    assert [x.value for x in v] == [640, 480, 0]
