"""numpy restatement of the Pillow-compatible on-device resize (include/b200_saber.h, b200_image_resize_pil_run):
torchvision's Resize(S) + CenterCrop on PIL images, i.e. Pillow's antialiased 8-bit BILINEAR resampler and a centre crop
whose offset rounds half to even. Coefficients are float64 steps that numpy never contracts into an FMA; the resampling
is exact integer arithmetic. tests/golden/pil_resize.json pins it to Pillow's bytes."""
import numpy as np

import image_resize_oracle as R

PRECISION_BITS = 22     # 32 - 8 - 2, Pillow's 8-bit coefficient precision


def geometry(h, w, resize_short, out_h, out_w):
    """(rh, rw, top, left) for the Pillow filter, or None where b200_image_resize_geometry_ex refuses: the reference
    filter's sizes, with torchvision CenterCrop's offsets round((r - out) / 2), half to even."""
    g = R.geometry(h, w, resize_short, out_h, out_w)
    if g is None:
        return None
    rh, rw, _, _ = g
    return rh, rw, round((rh - out_h) / 2), round((rw - out_w) / 2)


def vertical_first(h, w, rh):
    """Pillow's Image.resize runs the vertical pass first (as a resize of its own) for images more than 100 times
    taller than wide that shrink in height; every other image goes horizontal pass first."""
    return h > 100 * w and rh < h


def coeffs(in_size, out_size, coords):
    """(xmin, k) for output coordinates `coords` of an in_size -> out_size axis: Pillow's precompute_coeffs with the
    triangle filter (support 1), then normalize_coeffs_8bpc. k is int32 [len(coords), ksize], zero past each xmax."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 1.0 * fs
    ksize = 2 * int(np.ceil(support)) + 1
    ss = 1.0 / fs
    xmins, ks = [], np.zeros((len(coords), ksize), np.int32)
    for i, o in enumerate(coords):
        center = (o + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        wts = []
        for t in range(xmax):
            x = abs(((t + xmin) - center + 0.5) * ss)
            wts.append(1.0 - x if x < 1.0 else 0.0)
        ww = 0.0
        for v in wts:
            ww += v
        for t, v in enumerate(wts):
            v = v / ww if ww != 0.0 else v
            v = v * (1 << PRECISION_BITS)
            ks[i, t] = int(v - 0.5) if v < 0 else int(v + 0.5)
        xmins.append(xmin)
    return np.array(xmins, np.int64), ks


def _pass(src, axis, xmin, k):
    """One resampling pass along `axis` (0 rows, 1 columns) of uint8 src [h, w, c]: output i is
    clamp((2^21 + sum_t src[xmin_i + t] * k[i, t]) >> 22, 0, 255)."""
    s = np.moveaxis(src, axis, 0).astype(np.int64)
    idx = np.minimum(xmin[:, None] + np.arange(k.shape[1])[None, :], s.shape[0] - 1)    # k is 0 past xmax
    acc = np.full((len(xmin),) + s.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(k.shape[1]):
        acc += s[idx[:, t]] * k[:, t].reshape((-1,) + (1,) * (s.ndim - 1))
    assert np.abs(acc).max() < 2 ** 31
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize_u8(img_hwc, resize_short, out_h, out_w, vfirst=None):
    """uint8 [out_h, out_w, c]: the cropped window of Pillow's BILINEAR resize of img_hwc, only the needed rows and
    columns computed (each output depends only on its own taps). vfirst overrides the pass order."""
    img = np.asarray(img_hwc)
    h, w, _ = img.shape
    rh, rw, top, left = geometry(h, w, resize_short, out_h, out_w)
    ymin, ky = coeffs(h, rh, np.arange(out_h) + top)
    xmin, kx = coeffs(w, rw, np.arange(out_w) + left)
    if vertical_first(h, w, rh) if vfirst is None else vfirst:
        x0, x1 = xmin[0], xmin[-1] + kx.shape[1]
        tmp = _pass(img[:, x0:min(x1, w)], 0, ymin, ky)
        return _pass(tmp, 1, xmin - x0, kx)
    y0, y1 = ymin[0], ymin[-1] + ky.shape[1]
    tmp = _pass(img[y0:min(y1, h)], 1, xmin, kx)
    return _pass(tmp, 0, ymin - y0, ky)


def resize_batch(images, resize_short, out_h, out_w):
    return np.stack([resize_u8(im, resize_short, out_h, out_w) for im in images])


def pillow_resize(img_hwc, resize_short, out_h, out_w):
    """The same through Pillow (and torchvision for S > 0), for images of 1, 3 or 4 channels (L, RGB, CMYK)."""
    from PIL import Image
    img = np.asarray(img_hwc)
    c = img.shape[2]
    mode = {1: "L", 3: "RGB", 4: "CMYK"}[c]
    im = Image.frombytes(mode, (img.shape[1], img.shape[0]), np.ascontiguousarray(img).tobytes())
    if resize_short == 0:
        out = im.resize((out_w, out_h), Image.BILINEAR)
    else:
        import torchvision.transforms as T
        out = T.CenterCrop((out_h, out_w))(T.Resize(resize_short, T.InterpolationMode.BILINEAR)(im))
    a = np.asarray(out)
    return a.reshape(a.shape[0], a.shape[1], c)


# Images more than 100 times taller than wide, on both sides of Pillow's pass-order switch, as (h, w, out_h, out_w)
# stretches; the first eight go vertical first. The bytes of each differ between the two orders.
PASS_ORDER_CASES = [(2000, 16, 224, 224), (1800, 16, 224, 224), (3000, 16, 224, 224), (2000, 8, 224, 224),
                    (2000, 12, 224, 224), (2000, 16, 224, 100), (2000, 16, 100, 224), (1601, 16, 224, 224),
                    (1600, 16, 224, 224), (1500, 16, 224, 224), (1000, 16, 224, 224), (2000, 32, 224, 224),
                    (16, 2000, 224, 224), (500, 40, 224, 224)]

# (h, w, c, resize_short, out_h, out_w, image) of tests/golden/pil_resize.json (tools/make_pil_resize_golden.py)
GOLDEN_CASES = (
    [(h, w, 3, 256, 224, 224, "random") for h, w in
     [(375, 500), (480, 640), (1200, 1600), (300, 301), (100, 700), (224, 224), (200, 150), (257, 999)]]
    + [(3072, 4096, c, 0, 224, 224, "random") for c in (1, 3, 4)]
    + [(100, 150, 3, 0, 256, 384, "random"), (999, 333, 4, 0, 160, 200, "random"), (1, 1, 1, 0, 7, 5, "random"),
       (3024, 4032, 3, 256, 224, 224, "stripes"), (375, 500, 1, 232, 200, 160, "random"),
       (256, 339, 3, 256, 224, 224, "random"), (339, 256, 4, 256, 224, 224, "random")]
    + [(h, w, 3, 0, oh, ow, "random") for h, w, oh, ow in PASS_ORDER_CASES]
)


def case_image(h, w, c, image, seed):
    """uint8 [h, w, c]: uniform noise from `seed`, or vertical stripes of a 3.3-pixel period (antialiasing matters)."""
    if image == "stripes":
        x = np.arange(w)
        row = np.where((x * 10 // 33) % 2 == 0, 40, 230).astype(np.uint8)
        return np.ascontiguousarray(np.broadcast_to(row[None, :, None], (h, w, c)))
    return np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)
