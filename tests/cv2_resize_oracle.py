"""numpy restatement of OpenCV's INTER_LINEAR on-device resize (include/b200_saber.h, B200_IMAGE_RESIZE_CV2_LINEAR):
cv2.resize(img, (rw, rh)) with the default interpolation on 8-bit images, cropped with the reference filter's geometry
and floor offsets. The coefficients are numpy float64 / float32 steps, each rounded on its own; the sums are exact
integer arithmetic with OpenCV's shifts. NV12 / I420 frames and crop boxes reuse tests/yuv_oracle.py and
tests/crop_oracle.py. tests/golden/cv2_resize.json pins the restatement to the bytes of OpenCV 4.13 on x86-64
(tools/make_cv2_resize_golden.py).

No case is refused beyond the geometry's limits: the restatement equals cv2 on upscales and shrinks of either axis,
equal sizes and exact 2x shrinks, where cv2 switches to its area filter (for two channels the float one, which rounds
half to even)."""
import numpy as np

import crop_oracle as CR
import image_resize_oracle as R
import yuv_oracle as Y

COEF_BITS = 11          # INTER_RESIZE_COEF_BITS
COEF_SCALE = 1 << COEF_BITS


def geometry(h, w, resize_short, out_h, out_w):
    """(rh, rw, top, left), or None where b200_image_resize_geometry_ex refuses: the reference filter's."""
    return R.geometry(h, w, resize_short, out_h, out_w)


def axis(in_size, out_size, coords, columns):
    """(s0, s1, a0, a1) int64 arrays for output coordinates `coords` of an in_size -> out_size axis: taps and 11-bit
    weights. Columns clamp the taps and the fraction at the edges; rows clamp only the taps."""
    scale = 1.0 / (out_size / in_size)
    f = ((np.asarray(coords, np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if columns:
        lo = s < 0
        s, f = np.where(lo, 0, s), np.where(lo, np.float32(0), f)
        hi = s + 1 >= in_size
        s, f = np.where(hi, in_size - 1, s), np.where(hi, np.float32(0), f)
        s0, s1 = s, np.minimum(s + 1, in_size - 1)
    else:
        s0, s1 = np.clip(s, 0, in_size - 1), np.clip(s + 1, 0, in_size - 1)
    a0 = np.rint((np.float32(1) - f) * np.float32(COEF_SCALE)).astype(np.int64)
    a1 = np.rint(f * np.float32(COEF_SCALE)).astype(np.int64)
    return s0, s1, a0, a1


def resize_window(img_hwc, rh, rw, top, left, out_h, out_w):
    """uint8 [out_h, out_w, c]: rows [top, top + out_h) and columns [left, left + out_w) of cv2.resize(img, (rw, rh))."""
    img = np.asarray(img_hwc)
    h, w, c = img.shape
    y0, y1, b0, b1 = axis(h, rh, np.arange(out_h) + top, columns=False)
    x0, x1, a0, a1 = axis(w, rw, np.arange(out_w) + left, columns=True)
    p = img.astype(np.int64)
    a0, a1 = a0[None, :, None], a1[None, :, None]
    s0 = p[y0][:, x0] * a0 + p[y0][:, x1] * a1
    s1 = p[y1][:, x0] * a0 + p[y1][:, x1] * a1
    v = (((s0 >> 4) * b0[:, None, None]) >> 16) + (((s1 >> 4) * b1[:, None, None]) >> 16)
    assert v.min() >= 0 and v.max() <= 1020
    if c == 2 and h == 2 * rh and w == 2 * rw:
        out = (v + 1 + ((v >> 2) & 1)) >> 2         # the float area filter's half-to-even mean
    else:
        out = (v + 2) >> 2
    return out.astype(np.uint8)


def resize_u8(img_hwc, resize_short, out_h, out_w):
    """uint8 [out_h, out_w, c] of one image: the geometry, then the cropped window of the resize."""
    img = np.asarray(img_hwc)
    g = geometry(img.shape[0], img.shape[1], resize_short, out_h, out_w)
    assert g is not None, (img.shape, resize_short, out_h, out_w)
    return resize_window(img, *g, out_h, out_w)


def resize_batch(images, resize_short, out_h, out_w):
    return np.stack([resize_u8(im, resize_short, out_h, out_w) for im in images])


def resize_yuv(frame, fmt, resize_short, out_h, out_w):
    """uint8 [out_h, out_w, 3] of an NV12 / I420 frame: cvtColor, then the resize."""
    return resize_u8(Y.yuv_to_rgb(frame, fmt), resize_short, out_h, out_w)


def resize_boxes(frames, fmt, boxes, resize_short, out_h, out_w):
    """uint8 [len(boxes), out_h, out_w, c]: each box sliced out of its frame (converted first when YUV), then resized."""
    return np.stack([resize_u8(CR.crop(frames, fmt, b), resize_short, out_h, out_w) for b in boxes])


def cv2_resize(img_hwc, resize_short, out_h, out_w):
    """The same through OpenCV: cv2.resize to (rw, rh), then the crop."""
    import cv2
    img = np.asarray(img_hwc)
    rh, rw, top, left = geometry(img.shape[0], img.shape[1], resize_short, out_h, out_w)
    r = cv2.resize(img, (rw, rh), interpolation=cv2.INTER_LINEAR)
    return r.reshape(rh, rw, img.shape[2])[top:top + out_h, left:left + out_w]


def case_image(h, w, c, image, seed):
    """The source of a designed case: uint8 [h, w, c] uniform noise ("random") or all 255 ("white"); for "nv12" /
    "i420", a random frame of that format (c = 3)."""
    if image in Y.FORMATS:
        return Y.random_frame(h, w, Y.FORMATS[image], seed)
    if image == "white":
        return np.full((h, w, c), 255, np.uint8)
    return np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)


def case_resize(src, c, image, resize_short, out_h, out_w, cv2=False):
    """The restated (or, with cv2=True, OpenCV's) bytes of a designed case."""
    if image in Y.FORMATS:
        src = Y.cv2_rgb(src, Y.FORMATS[image]) if cv2 else Y.yuv_to_rgb(src, Y.FORMATS[image])
    return (cv2_resize if cv2 else resize_u8)(src, resize_short, out_h, out_w)


# (h, w, c, resize_short, out_h, out_w, image) of tests/golden/cv2_resize.json; case i uses seed i. Each axis up and
# down on its own and together; exact 2x shrinks for c = 1..4 (c = 2 rounds half to even) and with a crop; equal sizes,
# alone and under a crop; 1 x N, N x 1 and 1 x 1; output rows of 12 / 16 / 20 and 15 / 16 / 17 bytes around OpenCV's
# 16-byte vectors; a white image enlarged (the largest sums); short side + crop from 500 x 375 to 4032 x 3024 with even
# and odd margins; NV12 / I420 frames; and a 1 x 16384 stretch at the Net's limit.
GOLDEN_CASES = [
    (50, 224, 3, 0, 224, 224, "random"), (700, 224, 3, 0, 224, 224, "random"),
    (224, 60, 3, 0, 224, 224, "random"), (224, 700, 3, 0, 224, 224, "random"),
    (37, 41, 3, 0, 224, 224, "random"), (375, 500, 3, 0, 224, 224, "random"),
    (100, 700, 3, 0, 224, 224, "random"), (700, 100, 3, 0, 224, 224, "random"),
    (448, 448, 1, 0, 224, 224, "random"), (448, 448, 2, 0, 224, 224, "random"),
    (448, 448, 3, 0, 224, 224, "random"), (448, 448, 4, 0, 224, 224, "random"),
    (512, 600, 3, 256, 224, 224, "random"),
    (224, 224, 3, 0, 224, 224, "random"), (256, 300, 3, 256, 224, 224, "random"),
    (1, 500, 3, 0, 224, 224, "random"), (500, 1, 1, 0, 224, 224, "random"), (1, 1, 4, 0, 7, 5, "random"),
    (33, 47, 4, 0, 19, 3, "random"), (33, 47, 4, 0, 19, 4, "random"), (33, 47, 4, 0, 19, 5, "random"),
    (61, 29, 1, 0, 40, 15, "random"), (61, 29, 1, 0, 40, 16, "random"), (61, 29, 1, 0, 40, 17, "random"),
    (9, 13, 3, 0, 224, 224, "white"),
    (375, 500, 3, 256, 224, 224, "random"), (500, 375, 3, 232, 224, 224, "random"),
    (480, 640, 3, 256, 224, 224, "random"), (1080, 1920, 3, 256, 224, 224, "random"),
    (3024, 4032, 3, 256, 224, 224, "random"), (4032, 3024, 4, 256, 224, 224, "random"),
    (1080, 1920, 3, 256, 224, 224, "nv12"), (480, 640, 3, 232, 224, 224, "i420"),
    (2, 2, 3, 0, 224, 224, "nv12"), (720, 1280, 3, 0, 224, 224, "i420"), (448, 448, 3, 0, 224, 224, "nv12"),
    (1, 16384, 3, 0, 224, 224, "random"),
]
