"""numpy restatement of boxes cropped out of frames by the on-device resize (include/b200_saber.h,
b200_image_crop_resize_run): slice the box out of the frame (converted to RGB first for NV12 / I420), then apply the
existing restatements of the two filters to the slice. tests/test_cpu_image_crops.py pins it to Pillow, torchvision and
OpenCV."""
import numpy as np

import image_resize_oracle as R
import pil_resize_oracle as P
import yuv_oracle as Y

INTERLEAVED = 0
FORMATS = {"interleaved": INTERLEAVED, "nv12": Y.NV12, "i420": Y.I420}


def frame_rgb(frame, fmt):
    """uint8 [h, w, c] of a frame: itself when interleaved, its cvtColor when YUV."""
    return np.asarray(frame) if fmt == INTERLEAVED else Y.yuv_to_rgb(frame, fmt)


def crop(frames, fmt, box):
    """uint8 [height, width, c]: frame[top:top + height, left:left + width] of box (frame, top, left, height, width)."""
    f, t, l, h, w = (int(v) for v in box)
    img = frame_rgb(frames[f], fmt)
    assert 0 <= t and 0 <= l and h >= 1 and w >= 1 and t + h <= img.shape[0] and l + w <= img.shape[1], box
    return img[t:t + h, l:l + w]


def resize_box(frames, fmt, box, filt, resize_short, out_h, out_w):
    """uint8 [out_h, out_w, c] of one box with filter `filt` ("reference" or "pil")."""
    c = crop(frames, fmt, box)
    if filt == "pil":
        return P.resize_u8(c, resize_short, out_h, out_w)
    return R.image_resize_u8(c, resize_short, out_h, out_w)


def resize_boxes(frames, fmt, boxes, filt, resize_short, out_h, out_w):
    return np.stack([resize_box(frames, fmt, b, filt, resize_short, out_h, out_w) for b in boxes])


def frame_hw(frame, fmt):
    f = np.asarray(frame)
    return (f.shape[0], f.shape[1]) if fmt == INTERLEAVED else (f.shape[0] * 2 // 3, f.shape[1])


def random_frame(h, w, fmt, c, seed):
    if fmt == INTERLEAVED:
        return np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)
    return Y.random_frame(h, w, fmt, seed)


def designed_boxes(h, w, f=0):
    """Boxes of an h x w frame (h, w >= 8): a 1 x 1 box, the whole frame, a box touching each edge, and odd offsets
    and sizes."""
    return [(f, 0, 0, 1, 1), (f, h - 1, w - 1, 1, 1), (f, 0, 0, h, w), (f, 0, 1, 3, w - 2), (f, h - 5, 2, 5, 3),
            (f, 1, 0, h - 2, 5), (f, 3, w - 7, 4, 7), (f, 1, 3, h // 2 + 1, w // 2 + 1), (f, 3, 5, 7, 9)]


def outside_altered(frame, fmt, boxes):
    """The frame with every byte no box can read replaced: interleaved pixels outside every box inverted; for YUV the
    Y samples outside every box and the chroma samples whose whole 2 x 2 block lies outside every box (a block that
    straddles an odd box edge is read legitimately)."""
    f = np.array(frame, copy=True)
    if fmt == INTERLEAVED:
        keep = np.zeros(f.shape[:2], bool)
        for _, t, l, h, w in boxes:
            keep[t:t + h, l:l + w] = True
        f[~keep] = 255 - f[~keep]
        return f
    h, w = frame_hw(frame, fmt)
    y, u, v = (p.copy() for p in Y.planes(f, fmt))
    keep = np.zeros((h, w), bool)
    for _, t, l, bh, bw in boxes:
        keep[t:t + bh, l:l + bw] = True
    ckeep = keep.reshape(h // 2, 2, w // 2, 2).any(axis=(1, 3))
    y[~keep] = 255 - y[~keep]
    u[~ckeep] = 255 - u[~ckeep]
    v[~ckeep] = 255 - v[~ckeep]
    return Y.make_frame(y, u, v, fmt)
