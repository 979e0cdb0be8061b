"""numpy restatement of the YUV 4:2:0 sources of the on-device resize (include/b200_saber.h, b200_image_resize_yuv_run):
OpenCV's cvtColor(COLOR_YUV2RGB_NV12 / COLOR_YUV2RGB_I420), BT.601 limited range in 20-bit fixed point, and the
designed frames that pin it. A frame is OpenCV's 2-D layout, uint8 [h * 3 / 2, w]. tests/golden/yuv_resize.json pins
the restatement to cv2, Pillow and torchvision (tools/make_yuv_golden.py)."""
import numpy as np

import image_resize_oracle as R
import pil_resize_oracle as P

NV12, I420 = 1, 2
FORMATS = {"nv12": NV12, "i420": I420}


def planes(frame, fmt):
    """(Y [h, w], U [h/2, w/2], V [h/2, w/2]) of a frame."""
    f = np.asarray(frame)
    assert f.dtype == np.uint8 and f.ndim == 2 and f.shape[0] % 3 == 0
    h, w = f.shape[0] * 2 // 3, f.shape[1]
    assert h % 2 == 0 and w % 2 == 0, (h, w)
    y = f[:h]
    if fmt == NV12:
        uv = f[h:].reshape(h // 2, w // 2, 2)
        return y, uv[..., 0], uv[..., 1]
    c = f[h:].reshape(-1)
    n = (h // 2) * (w // 2)
    return y, c[:n].reshape(h // 2, w // 2), c[n:].reshape(h // 2, w // 2)


def make_frame(y, u, v, fmt):
    """The frame of planes Y [h, w], U and V [h/2, w/2] in `fmt`."""
    h, w = y.shape
    if fmt == NV12:
        chroma = np.stack([u, v], axis=-1).reshape(h // 2, w)
    else:
        chroma = np.concatenate([u.reshape(-1), v.reshape(-1)]).reshape(h // 2, w)
    return np.ascontiguousarray(np.concatenate([y, chroma]).astype(np.uint8))


def convert(y, u, v):
    """uint8 R, G, B of (Y, U, V) arrays of one shape: the fixed-point arithmetic of the header, in int64."""
    yy = np.maximum(y.astype(np.int64) - 16, 0) * 1220542 + (1 << 19)
    u = u.astype(np.int64) - 128
    v = v.astype(np.int64) - 128
    r = (yy + 1673527 * v) >> 20
    g = (yy - 852492 * v - 409993 * u) >> 20
    b = (yy + 2116026 * u) >> 20
    return np.stack([np.clip(c, 0, 255) for c in (r, g, b)], axis=-1).astype(np.uint8)


def yuv_to_rgb(frame, fmt):
    """uint8 [h, w, 3] R, G, B of a frame: pixel (y, x) takes chroma sample (y/2, x/2)."""
    y, u, v = planes(frame, fmt)
    up = lambda c: np.repeat(np.repeat(c, 2, axis=0), 2, axis=1)      # noqa: E731
    return convert(y, up(u), up(v))


def resize(frame, fmt, filt, resize_short, out_h, out_w):
    """uint8 [out_h, out_w, 3]: the conversion, then the resize and crop of filter `filt` ("reference" or "pil")."""
    rgb = yuv_to_rgb(frame, fmt)
    if filt == "pil":
        return P.resize_u8(rgb, resize_short, out_h, out_w)
    return R.image_resize_u8(rgb, resize_short, out_h, out_w)


def resize_batch(frames, fmt, filt, resize_short, out_h, out_w):
    return np.stack([resize(f, fmt, filt, resize_short, out_h, out_w) for f in frames])


def random_frame(h, w, fmt, seed):
    """A frame of uniform random bytes (every plane)."""
    rng = np.random.default_rng(seed)
    return make_frame(rng.integers(0, 256, (h, w), dtype=np.uint8), rng.integers(0, 256, (h // 2, w // 2), np.uint8),
                      rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8), fmt)


EXHAUSTIVE = 4096


def exhaustive_planes():
    """Planes of a 4096 x 4096 frame holding every (Y, U, V) triple once: chroma block b (row-major over 2048 x 2048)
    has U = (b // 64) >> 8, V = (b // 64) & 255 and the four lumas 4 * (b % 64) + 0..3 in its 2 x 2 pixels."""
    n = EXHAUSTIVE // 2
    b = np.arange(n * n, dtype=np.int64)
    u = ((b // 64) >> 8).astype(np.uint8).reshape(n, n)
    v = ((b // 64) & 255).astype(np.uint8).reshape(n, n)
    base = (4 * (b % 64)).reshape(n, n)
    y = np.empty((EXHAUSTIVE, EXHAUSTIVE), np.uint8)
    y[0::2, 0::2], y[0::2, 1::2] = base, base + 1
    y[1::2, 0::2], y[1::2, 1::2] = base + 2, base + 3
    return y, u, v


def exhaustive_frame(fmt):
    return make_frame(*exhaustive_planes(), fmt)


# (h, w, resize_short, out_h, out_w) of tests/golden/yuv_resize.json, each in both formats: the smallest frame, 1080p
# and 2160p at S = 256 and 232, an odd rw - W (half-even crop), a 2000 x 16 frame on the vertical-first side of
# Pillow's pass-order switch and a 1600 x 16 one on the other side, and a stretch
GOLDEN_CASES = [(2, 2, 256, 224, 224), (1080, 1920, 256, 224, 224), (1080, 1920, 232, 224, 224),
                (2160, 3840, 256, 224, 224), (2160, 3840, 232, 224, 224), (480, 640, 256, 224, 224),
                (2000, 16, 0, 224, 224), (1600, 16, 0, 224, 224), (720, 1280, 0, 224, 224)]


def golden_frame(h, w, fmt, index):
    return random_frame(h, w, fmt, seed=1000 + index)


def cv2_rgb(frame, fmt):
    import cv2
    return cv2.cvtColor(frame, cv2.COLOR_YUV2RGB_NV12 if fmt == NV12 else cv2.COLOR_YUV2RGB_I420)
