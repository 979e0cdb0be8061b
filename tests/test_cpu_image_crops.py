"""CPU suite: boxes cropped out of frames by the on-device resize (include/b200_saber.h, b200_image_crop_resize_run).
The restatement (tests/crop_oracle.py: slicing plus the existing filter restatements) against Pillow's crop with
torchvision's Resize / CenterCrop and resized_crop, and against OpenCV's cvtColor followed by slicing; the crop entry's
layout; the entry point's argument checks without a GPU; the Python box checks."""
import ctypes as C

import numpy as np
import pytest

import crop_oracle as K
import yuv_oracle as Y


def _pillow_crop(img, box, resize_short, out_h, out_w):
    """torchvision on a PIL image: CenterCrop((H, W))(Resize(S)(img.crop(...))), or resized_crop when S = 0."""
    from PIL import Image
    import torchvision.transforms as T
    import torchvision.transforms.functional as F
    _, t, l, h, w = box
    c = img.shape[2]
    im = Image.frombytes({1: "L", 3: "RGB", 4: "CMYK"}[c], (img.shape[1], img.shape[0]),
                         np.ascontiguousarray(img).tobytes())
    if resize_short == 0:
        out = F.resized_crop(im, t, l, h, w, [out_h, out_w], T.InterpolationMode.BILINEAR)
    else:
        out = T.CenterCrop((out_h, out_w))(T.Resize(resize_short, T.InterpolationMode.BILINEAR)(
            im.crop((l, t, l + w, t + h))))
    a = np.asarray(out)
    return a.reshape(a.shape[0], a.shape[1], c)


@pytest.mark.parametrize("s", [0, 232, 256])
@pytest.mark.parametrize("c", [1, 3, 4])
def test_pil_restatement_equals_torchvision_on_designed_boxes(c, s):
    pytest.importorskip("torchvision")
    frame = K.random_frame(61, 83, K.INTERLEAVED, c, seed=10 * c + s)
    for box in K.designed_boxes(61, 83):
        want = _pillow_crop(frame, box, s, 224, 224)
        got = K.resize_box([frame], K.INTERLEAVED, box, "pil", s, 224, 224)
        assert np.array_equal(got, want), box


@pytest.mark.parametrize("box, frame_hw", [((0, 50, 7, 2000, 16), (2100, 40)), ((0, 3, 11, 1600, 16), (1700, 40))])
def test_pass_order_is_judged_on_the_box(box, frame_hw):
    """A 2000 x 16 box goes vertical first and a 1600 x 16 one horizontal first, while neither frame is tall enough
    for the switch: Pillow decides on the cropped image, and so does the restatement."""
    pytest.importorskip("torchvision")
    import pil_resize_oracle as P
    frame = K.random_frame(*frame_hw, K.INTERLEAVED, 3, seed=box[3])
    assert not P.vertical_first(frame_hw[0], frame_hw[1], 224)
    assert P.vertical_first(box[3], box[4], 224) == (box[3] == 2000)
    got = K.resize_box([frame], K.INTERLEAVED, box, "pil", 0, 224, 224)
    assert np.array_equal(got, _pillow_crop(frame, box, 0, 224, 224))
    # the other pass order gives other bytes, so the comparison above tells the orders apart
    other = P.resize_u8(K.crop([frame], K.INTERLEAVED, box), 0, 224, 224, vfirst=box[3] != 2000)
    assert not np.array_equal(got, other)


@pytest.mark.parametrize("name", ["nv12", "i420"])
def test_yuv_box_equals_cvtcolor_then_slicing(name):
    cv2 = pytest.importorskip("cv2")
    fmt = Y.FORMATS[name]
    frame = Y.random_frame(40, 58, fmt, seed=fmt)
    rgb = cv2.cvtColor(frame, cv2.COLOR_YUV2RGB_NV12 if fmt == Y.NV12 else cv2.COLOR_YUV2RGB_I420)
    for box in K.designed_boxes(40, 58) + [(0, 1, 1, 1, 1), (0, 7, 9, 3, 5), (0, 0, 57, 40, 1)]:
        _, t, l, h, w = box
        assert np.array_equal(K.crop([frame], fmt, box), rgb[t:t + h, l:l + w]), box


@pytest.mark.parametrize("name", ["nv12", "i420"])
def test_yuv_box_through_pillow(name):
    """cvtColor + Pillow crop + torchvision on odd boxes of a YUV frame equal the restatement."""
    cv2 = pytest.importorskip("cv2")
    pytest.importorskip("torchvision")
    fmt = Y.FORMATS[name]
    frame = Y.random_frame(120, 90, fmt, seed=7 + fmt)
    rgb = cv2.cvtColor(frame, cv2.COLOR_YUV2RGB_NV12 if fmt == Y.NV12 else cv2.COLOR_YUV2RGB_I420)
    for s in (0, 232):
        for box in [(0, 3, 5, 77, 41), (0, 1, 0, 119, 89), (0, 0, 1, 1, 1)]:
            assert np.array_equal(K.resize_box([frame], fmt, box, "pil", s, 224, 224),
                                  _pillow_crop(rgb, box, s, 224, 224)), (s, box)


def test_outside_altered_keeps_exactly_what_a_box_reads():
    fmt = Y.NV12
    frame = Y.random_frame(8, 8, fmt, 1)
    boxes = [(0, 1, 1, 3, 2)]                    # rows 1..3, columns 1..2: chroma blocks (0..1, 0..1)
    alt = K.outside_altered(frame, fmt, boxes)
    y0, u0, _ = Y.planes(frame, fmt)
    y1, u1, _ = Y.planes(alt, fmt)
    assert np.array_equal(y0[1:4, 1:3], y1[1:4, 1:3]) and (y0 != y1).sum() == 64 - 6
    assert np.array_equal(u0[:2, :2], u1[:2, :2]) and (u0 != u1).sum() == 16 - 4
    assert np.array_equal(K.crop([alt], fmt, boxes[0]), K.crop([frame], fmt, boxes[0]))


def test_crop_entry_layout():
    from anakin_b200 import saber_abi as A
    assert C.sizeof(A.ImageCropEntry) == 48 and C.sizeof(A.ImageResizeEntry) == 32
    assert A.ImageCropEntry.r.offset == 0
    assert [getattr(A.ImageCropEntry, f).offset for f in ("frame_h", "frame_w", "box_top", "box_left")] == [32, 36, 40, 44]


def _desc(A, n=2, c=3, oh=224, ow=224):
    d = A.ImageResizeDesc()
    d.n, d.c, d.out_h, d.out_w = n, c, oh, ow
    return d


def test_crop_run_validates_arguments_without_a_gpu():
    from anakin_b200 import saber_abi as A
    lib = A.load()
    run = lib.b200_image_crop_resize_run
    p = C.c_void_p(16)      # never dereferenced: argument errors are reported before any device work
    good = _desc(A)
    for filt in (0, 1):
        for fmt in (A.IMAGE_INTERLEAVED, A.IMAGE_YUV_NV12, A.IMAGE_YUV_I420):
            assert run(None, filt, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
            for i in range(3 + filt):       # src, table, out; and the workspace for the Pillow filter
                a = [p, p, p, p]
                a[[0, 1, 3, 2][i]] = None
                assert run(C.byref(good), filt, fmt, 500, 500, 256, *a, None) == A.INVALID_VALUE, (filt, fmt, i)
            for d in (_desc(A, n=0), _desc(A, oh=0), _desc(A, ow=0), _desc(A, c=5)):
                assert run(C.byref(d), filt, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
        for fmt in (-1, 3):
            assert run(C.byref(good), filt, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
        for fmt in (A.IMAGE_YUV_NV12, A.IMAGE_YUV_I420):
            for c in (1, 2, 4):
                assert run(C.byref(_desc(A, c=c)), filt, fmt, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
    for filt in (-1, 2):
        assert run(C.byref(good), filt, 0, 500, 500, 256, p, p, p, p, None) == A.INVALID_VALUE
    for mh, mw, s in ((0, 500, 256), (500, 500, -1), (500, 500, 100)):
        assert run(C.byref(good), 1, 0, mh, mw, s, p, p, p, p, None) == A.INVALID_VALUE


def test_python_box_checks():
    from anakin_b200 import api
    assert api.pack_boxes([[0, 1, 2, 3, 4]]).dtype == np.int32
    assert api.pack_boxes(np.array([[0, 1, 2, 3, 4]], np.uint8)).tolist() == [[0, 1, 2, 3, 4]]
    for bad in ([0, 1, 2, 3, 4], np.zeros((2, 4), np.int32), np.zeros((0, 5), np.int32), np.zeros((1, 5, 1), np.int32)):
        with pytest.raises(api.AnakinError, match="boxes: a \\[k, 5\\] array"):
            api.pack_boxes(bad)
    for bad in (np.zeros((1, 5), np.float32), [[0, 1, 2, 3.5, 4]], np.zeros((1, 5), bool)):
        with pytest.raises(api.AnakinError, match="boxes: integer pixel coordinates expected"):
            api.pack_boxes(bad)
    with pytest.raises(api.AnakinError, match="outside int32"):
        api.pack_boxes(np.array([[0, 0, 0, 1, 2 ** 40]], np.int64))
