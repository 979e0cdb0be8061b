"""numpy restatement of the on-device image resize (include/b200_saber.h, b200_image_resize_run): the geometry, the
reference's BILINEAR_NO_ALIGN arithmetic (x86 saber_resize.cpp, resize_bilinear_no_align_kernel) evaluated at the
cropped pixels, and the rounding to 8 bits. Every float operation is numpy float32 or float64 arithmetic, which never
contracts into an FMA, so it is the reference's result bit for bit (tests/golden/ref_resize.json pins it)."""
import numpy as np

MAX_RESIZED = 1 << 23


def geometry(h, w, resize_short, out_h, out_w):
    """(rh, rw, top, left) of an h x w image, or None where b200_image_resize_geometry returns B200_INVALID_VALUE."""
    if min(h, w, out_h, out_w) < 1 or max(h, w) > MAX_RESIZED or resize_short < 0:
        return None
    if resize_short == 0:
        rh, rw = out_h, out_w
    else:
        if resize_short < max(out_h, out_w):
            return None
        if h <= w:
            rh, rw = resize_short, resize_short * w // h
        else:
            rh, rw = resize_short * h // w, resize_short
    if rh > MAX_RESIZED or rw > MAX_RESIZED:
        return None
    return rh, rw, (rh - out_h) // 2, (rw - out_w) // 2


def _axis(size, resized, coords):
    """Source taps and fraction along one axis for resized coordinates `coords` (the reference's fw / fh)."""
    scale = np.float32(size) / np.float32(resized)
    f = scale * (coords.astype(np.float32) + np.float32(0.5)) - np.float32(0.5)
    f = np.where(f < 0, np.float32(0), f).astype(np.float32)
    i0 = f.astype(np.int64)
    i1 = i0 + (i0 < size - 1)
    return i0, i1, (f - i0.astype(np.float32)).astype(np.float32)


def resize_bilinear_float(img_hwc, rh, rw, top, left, out_h, out_w):
    """fp32 [out_h, out_w, c]: the reference's resize of img_hwc to rh x rw, rows top.., columns left.."""
    h, w, _ = img_hwc.shape
    y0, y1, fh = _axis(h, rh, np.arange(out_h) + top)
    x0, x1, fw = _axis(w, rw, np.arange(out_w) + left)
    fh64, fw64 = fh.astype(np.float64)[:, None], fw.astype(np.float64)[None, :]
    w00 = ((1.0 - fh64) * (1.0 - fw64)).astype(np.float32)[..., None]
    w01 = (fw64 * (1.0 - fh64)).astype(np.float32)[..., None]
    w10 = (fh64 * (1.0 - fw64)).astype(np.float32)[..., None]
    w11 = (fw[None, :] * fh[:, None]).astype(np.float32)[..., None]      # float x float in the reference
    p = img_hwc.astype(np.float32)
    r0, r1 = p[y0], p[y1]
    v = w00 * r0[:, x0] + w01 * r0[:, x1]
    v = v + w10 * r1[:, x0]
    v = v + w11 * r1[:, x1]
    assert v.dtype == np.float32
    return v


def image_resize_u8(img_hwc, resize_short, out_h, out_w, return_float=False):
    """uint8 [out_h, out_w, c] the kernel writes for one image (saturate(rint(v)), half to even); with return_float
    also the fp32 stage."""
    img_hwc = np.asarray(img_hwc)
    assert img_hwc.dtype == np.uint8 and img_hwc.ndim == 3
    g = geometry(img_hwc.shape[0], img_hwc.shape[1], resize_short, out_h, out_w)
    if g is None:
        raise ValueError("no valid resize geometry for %s, resize_short %d, %d x %d" %
                         (img_hwc.shape, resize_short, out_h, out_w))
    v = resize_bilinear_float(img_hwc, *g, out_h, out_w)
    u8 = np.clip(np.rint(v), 0, 255).astype(np.uint8)
    return (u8, v) if return_float else u8


def resize_batch(images, resize_short, out_h, out_w):
    """uint8 [n, out_h, out_w, c] of a request (the image input tensor after the ImageResize op)."""
    return np.stack([image_resize_u8(a, resize_short, out_h, out_w) for a in images])


# The cases pinned against the reference's own function (tests/golden/ref_resize.json, tools/make_ref_resize_golden.py):
# (h, w, c, resize_short, out_h, out_w, seed)
REF_CASES = [
    (375, 500, 3, 256, 224, 224, 1),     # ImageNet-typical landscape, non-integer downscale
    (500, 375, 3, 256, 224, 224, 2),     # portrait
    (448, 448, 3, 0, 224, 224, 3),       # exact 2x downscale
    (960, 1280, 3, 256, 224, 224, 4),    # large non-integer downscale
    (100, 150, 3, 256, 224, 224, 5),     # upscale
    (16, 1000, 3, 256, 224, 224, 6),     # extreme aspect ratio (resized 256 x 16000)
    (1, 1, 3, 0, 224, 224, 7),           # one pixel
    (224, 224, 4, 0, 224, 224, 8),       # identity
    (333, 517, 1, 232, 200, 160, 9),     # odd margins, one channel
    (37, 53, 4, 0, 200, 160, 10),        # stretch upscale, four channels
]


def ref_case_image(case):
    h, w, c, _, _, _, seed = case
    return np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)


def ref_case_key(case):
    return "resize_%dx%dx%d_s%d_%dx%d" % case[:6]
