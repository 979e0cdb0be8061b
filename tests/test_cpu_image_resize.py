"""On-device image resize without a GPU: the geometry entry point against the numpy restatement, the argument checks of
the kernel's entry point (made before the device check), the numpy oracle against the reference's own resize (digests
in tests/golden/ref_resize.json) and against OpenCV, and the Graph attributes with their rejections."""
import ctypes as C
import hashlib
import json
import os
import tempfile

import numpy as np
import pytest

import image_resize_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FMT = {"mean": [123.675, 116.28, 103.53], "scale": [1 / 58.395, 1 / 57.12, 1 / 57.375], "src_channel": [2, 1, 0]}


def _geometry(lib, h, w, s, oh, ow):
    out = [C.c_int32(-7) for _ in range(4)]
    rc = lib.b200_image_resize_geometry(h, w, s, oh, ow, *[C.byref(x) for x in out])
    return rc, tuple(x.value for x in out)


def test_geometry_matches_the_numpy_restatement():
    from anakin_b200 import saber_abi as A
    lib = A.load()
    sides = [1, 2, 3, 15, 16, 100, 223, 224, 225, 231, 255, 256, 257, 333, 375, 500, 517, 960, 1000, 1280, 16384]
    cases = [(h, w, s, oh, ow) for h in sides for w in sides for s in (0, 224, 232, 256, 300)
             for oh, ow in ((224, 224), (200, 160))]
    cases += [
        (1, 1 << 23, 1, 1, 1),                   # rw exactly 2^23
        (1, (1 << 23) + 1, 0, 224, 224),         # source side past 2^23
        (2, 1 << 23, 256, 224, 224),             # rw = 2^30: rejected
        (16, 1000, 256, 224, 224),               # rw = 16000
        (16384, 1, 256, 224, 224),               # rh = 4,194,304
        (16384, 1, 600, 224, 224),               # rh = 9,830,400 > 2^23: rejected
        (100, 100, 223, 224, 224),               # 0 < S < max(H, W)
        (100, 100, 224, 224, 200),
        (100, 100, -1, 224, 224),
        (0, 100, 0, 224, 224), (100, 0, 0, 224, 224), (100, 100, 0, 0, 224), (100, 100, 0, 224, 0),
        (101, 100, 256, 224, 224), (100, 101, 256, 224, 224),    # odd margins
    ]
    for case in cases:
        want = O.geometry(*case)
        rc, got = _geometry(lib, *case)
        if want is None:
            assert rc == A.INVALID_VALUE, (case, rc, got)
        else:
            assert rc == A.SUCCESS and got == want, (case, rc, got, want)
    assert O.geometry(1, 1 << 23, 1, 1, 1) == (1, 1 << 23, 0, ((1 << 23) - 1) // 2)
    assert O.geometry(2, 1 << 23, 256, 224, 224) is None
    # null outputs
    z = C.c_int32()
    assert lib.b200_image_resize_geometry(10, 10, 0, 4, 4, None, C.byref(z), C.byref(z), C.byref(z)) == A.INVALID_VALUE


def test_resize_run_validates_without_a_gpu():
    from anakin_b200 import saber_abi as A
    lib = A.load()
    buf = (C.c_uint8 * 256)()
    p = C.cast(buf, C.c_void_p)

    def desc(n=1, c=3, oh=4, ow=4):
        d = A.ImageResizeDesc()
        d.n, d.c, d.out_h, d.out_w = n, c, oh, ow
        return d
    for bad in (desc(n=0), desc(c=0), desc(c=5), desc(oh=0), desc(ow=0), desc(n=-1)):
        assert lib.b200_image_resize_run(C.byref(bad), p, p, p, None) == A.INVALID_VALUE
    good = desc()
    assert lib.b200_image_resize_run(None, p, p, p, None) == A.INVALID_VALUE
    assert lib.b200_image_resize_run(C.byref(good), None, p, p, None) == A.INVALID_VALUE
    assert lib.b200_image_resize_run(C.byref(good), p, None, p, None) == A.INVALID_VALUE
    assert lib.b200_image_resize_run(C.byref(good), p, p, None, None) == A.INVALID_VALUE
    assert C.sizeof(A.ImageResizeEntry) == 32


def _digest(a):
    a = np.ascontiguousarray(a)
    return [list(a.shape), str(a.dtype), hashlib.sha256(a.tobytes()).hexdigest()]


def test_oracle_float_stage_equals_the_reference_resize():
    with open(os.path.join(HERE, "golden", "ref_resize.json")) as f:
        ref = json.load(f)
    assert len(O.REF_CASES) >= 8
    for case in O.REF_CASES:
        _, v = O.image_resize_u8(O.ref_case_image(case), case[3], case[4], case[5], return_float=True)
        assert _digest(v) == ref[O.ref_case_key(case)], case


def test_oracle_is_the_identity_at_the_network_size():
    for c in (1, 3, 4):
        img = np.random.default_rng(c).integers(0, 256, (224, 224, c), dtype=np.uint8)
        assert np.array_equal(O.image_resize_u8(img, 0, 224, 224), img)
        img = img[:200, :160]
        assert np.array_equal(O.image_resize_u8(img, 0, 200, 160), img)


@pytest.mark.parametrize("h,w,c,s,oh,ow", [(375, 500, 3, 256, 224, 224), (500, 375, 3, 256, 224, 224),
                                           (960, 1280, 3, 256, 224, 224), (100, 150, 3, 256, 224, 224),
                                           (448, 448, 3, 0, 224, 224), (333, 517, 1, 232, 200, 160),
                                           (37, 53, 4, 0, 200, 160), (480, 640, 3, 232, 224, 224)])
def test_oracle_within_one_of_opencv(h, w, c, s, oh, ow):
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(h * w + c).integers(0, 256, (h, w, c), dtype=np.uint8)
    rh, rw, top, left = O.geometry(h, w, s, oh, ow)
    r = cv2.resize(img, (rw, rh), interpolation=cv2.INTER_LINEAR)
    if r.ndim == 2:
        r = r[..., None]
    want = r[top:top + oh, left:left + ow]
    got = O.image_resize_u8(img, s, oh, ow)
    assert np.abs(got.astype(int) - want.astype(int)).max() <= 1


def _graph(model="tiny_resnet"):
    from anakin_b200 import anakin_bin, api, modelzoo
    return api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build(model, 1)))


def test_resize_attributes_survive_save_load_reshape_and_reset_batch_size():
    from anakin_b200 import api
    G = _graph()
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    assert G.input_image_resize("input_0") is None
    G.set_input_image_resize("input_0", 1280, 960, 256)
    want = {"max_h": 1280, "max_w": 960, "resize_short": 256}
    assert G.input_image_resize("input_0") == want
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        G2 = api.Graph.from_file(p)
    assert G2.input_image_resize("input_0") == want
    assert G2.input_image("input_0") is not None
    G2.ResetBatchSize("input_0", 8)
    G2.Reshape("input_0", [8, 3, 40, 48])
    G2.Optimize()
    assert G2.input_image_resize("input_0") == want
    G2.set_input_image_resize("input_0", 16384, 1, 0)          # the bounds are inclusive; 0 = stretch
    assert G2.input_image_resize("input_0") == {"max_h": 16384, "max_w": 1, "resize_short": 0}


def test_set_input_image_resize_rejections_python():
    from anakin_b200 import api
    G = _graph()
    with pytest.raises(api.AnakinError, match="not an image input"):
        G.set_input_image_resize("input_0", 500, 500, 256)       # set_input_image first
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    with pytest.raises(api.AnakinError, match="not an Input"):
        G.set_input_image_resize("conv1", 500, 500, 256)
    with pytest.raises(api.AnakinError, match="no node"):
        G.set_input_image_resize("no_such_input", 500, 500, 256)
    for mh, mw in ((0, 500), (500, 0), (16385, 500), (500, 16385), (-1, 500)):
        with pytest.raises(api.AnakinError, match="1..16384"):
            G.set_input_image_resize("input_0", mh, mw, 256)
    with pytest.raises(api.AnakinError, match="resize_short"):
        G.set_input_image_resize("input_0", 500, 500, -1)
    assert G.input_image_resize("input_0") is None, "a rejected call must leave the input as it was"


def test_set_input_image_resize_rejections_c_api():
    from anakin_b200 import api
    lib = api.load()
    G = _graph()
    h = G._h
    assert lib.anakin_graph_set_input_image_resize(h, b"input_0", 500, 500, 256) != 0
    assert b"not an image input" in lib.anakin_last_error()
    G.set_input_image("input_0", FMT["mean"], FMT["scale"], FMT["src_channel"])
    for args, msg in (((b"conv1", 500, 500, 256), b"not an Input"), ((b"nope", 500, 500, 256), b"no node"),
                      ((b"input_0", 0, 500, 256), b"1..16384"), ((b"input_0", 500, 16385, 256), b"1..16384"),
                      ((b"input_0", 500, 500, -3), b"resize_short")):
        assert lib.anakin_graph_set_input_image_resize(h, *args) != 0, args
        assert msg in lib.anakin_last_error(), (args, lib.anakin_last_error())
    assert lib.anakin_graph_set_input_image_resize(h, None, 500, 500, 256) != 0
    assert lib.anakin_graph_set_input_image_resize(None, b"input_0", 500, 500, 256) != 0
    v = [C.c_int(-5) for _ in range(3)]
    assert lib.anakin_graph_input_image_resize(h, b"input_0", *[C.byref(x) for x in v]) == 0
    assert lib.anakin_graph_set_input_image_resize(h, b"input_0", 640, 480, 0) == 0
    assert lib.anakin_graph_input_image_resize(h, b"input_0", *[C.byref(x) for x in v]) == 1
    assert [x.value for x in v] == [640, 480, 0]
    assert lib.anakin_graph_input_image_resize(h, b"input_0", None, None, None) == 1


def test_pack_images_layout():
    from anakin_b200 import api
    a = np.arange(2 * 3 * 3, dtype=np.uint8).reshape(2, 3, 3)
    b = np.arange(4 * 1 * 3, dtype=np.uint8).reshape(4, 1, 3) + 100
    pix, hw = api.pack_images([a, b])
    assert hw.dtype == np.int32 and hw.tolist() == [[2, 3], [4, 1]]
    assert np.array_equal(pix, np.concatenate([a.ravel(), b.ravel()]))
    with pytest.raises(api.AnakinError):
        api.pack_images([a.astype(np.float32)])
    with pytest.raises(api.AnakinError):
        api.pack_images([a[..., 0]])
