"""numpy restatement of Pillow's BICUBIC on-device resize (include/b200_saber.h, B200_IMAGE_RESIZE_PIL_BICUBIC):
torchvision's Resize(S, interpolation=BICUBIC) + CenterCrop on PIL images. Pillow runs BICUBIC through the same
precompute_coeffs, normalize_coeffs_8bpc and two 8-bit passes as BILINEAR, so this module takes the geometry, the
pass-order rule and the designed cases from tests/pil_resize_oracle.py and changes only the filter: the cubic
convolution of a = -0.5 with support 2, read at x / filterscale. Coefficients are float64 steps that numpy never
contracts into an FMA; the resampling is exact integer arithmetic. tests/golden/pil_bicubic_resize.json pins it to the
bytes of x86-64 Pillow, which evaluates the filter without contraction either (a build that contracts can differ in
the last bit of a weight)."""
import numpy as np

import pil_resize_oracle as P

PRECISION_BITS = P.PRECISION_BITS
SUPPORT = 2.0           # the cubic's support at scale 1 (the triangle's is 1)


def cubic(x):
    """Pillow's bicubic_filter with a = -0.5, in its order of operations."""
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def kmax(in_max, out_min, support=SUPPORT):
    """The tap bound of b200_image_resize_workspace for one axis: 2 * ceil(f * in_max / out_min) + 1 for the filter's
    support f (2 for BICUBIC, 1 for BILINEAR), at least 2 * f + 1."""
    f = int(support)
    return 2 * max(-(-f * in_max // out_min), f) + 1


def coeffs(in_size, out_size, coords):
    """(xmin, k) for output coordinates `coords` of an in_size -> out_size axis: Pillow's precompute_coeffs with the
    cubic filter, then normalize_coeffs_8bpc. k is int32 [len(coords), ksize], zero past each xmax."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = SUPPORT * fs
    ksize = 2 * int(np.ceil(support)) + 1
    ss = 1.0 / fs                       # not 1 / support: the filter reads x / filterscale
    xmins, ks = [], np.zeros((len(coords), ksize), np.int32)
    for i, o in enumerate(coords):
        center = (o + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        wts = [cubic(((t + xmin) - center + 0.5) * ss) for t in range(xmax)]
        ww = 0.0
        for v in wts:
            ww += v
        for t, v in enumerate(wts):
            v = v / ww if ww != 0.0 else v
            v = v * (1 << PRECISION_BITS)
            ks[i, t] = int(v - 0.5) if v < 0 else int(v + 0.5)
        xmins.append(xmin)
    return np.array(xmins, np.int64), ks


def _pass(src, axis, xmin, k, sums):
    """One resampling pass along `axis` (0 rows, 1 columns) of uint8 src [h, w, c]: output i is
    clamp((2^21 + sum_t src[xmin_i + t] * k[i, t]) >> 22, 0, 255). sums, a list or None, receives the accumulators."""
    s = np.moveaxis(src, axis, 0).astype(np.int64)
    idx = np.minimum(xmin[:, None] + np.arange(k.shape[1])[None, :], s.shape[0] - 1)    # k is 0 past xmax
    acc = np.full((len(xmin),) + s.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(k.shape[1]):
        acc += s[idx[:, t]] * k[:, t].reshape((-1,) + (1,) * (s.ndim - 1))
    assert np.abs(acc).max() < 2 ** 31
    if sums is not None:
        sums.append(acc)
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize_u8(img_hwc, resize_short, out_h, out_w, vfirst=None, sums=None):
    """uint8 [out_h, out_w, c]: the cropped window of Pillow's BICUBIC resize of img_hwc, only the needed rows and
    columns computed. vfirst overrides the pass order; sums, a list, receives the two passes' int32 accumulators
    (2^21 + sum), first pass first."""
    img = np.asarray(img_hwc)
    h, w, _ = img.shape
    rh, rw, top, left = P.geometry(h, w, resize_short, out_h, out_w)
    ymin, ky = coeffs(h, rh, np.arange(out_h) + top)
    xmin, kx = coeffs(w, rw, np.arange(out_w) + left)
    if P.vertical_first(h, w, rh) if vfirst is None else vfirst:
        x0, x1 = xmin[0], xmin[-1] + kx.shape[1]
        tmp = _pass(img[:, x0:min(x1, w)], 0, ymin, ky, sums)
        return _pass(tmp, 1, xmin - x0, kx, sums)
    y0, y1 = ymin[0], ymin[-1] + ky.shape[1]
    tmp = _pass(img[y0:min(y1, h)], 1, xmin, kx, sums)
    return _pass(tmp, 0, ymin - y0, ky, sums)


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
        out = im.resize((out_w, out_h), Image.BICUBIC)
    else:
        import torchvision.transforms as T
        out = T.CenterCrop((out_h, out_w))(T.Resize(resize_short, T.InterpolationMode.BICUBIC)(im))
    a = np.asarray(out)
    return a.reshape(a.shape[0], a.shape[1], c)


def case_image(h, w, c, image, seed):
    """uint8 [h, w, c]: the images of pil_resize_oracle.case_image, or "checker", a 0 / 255 checkerboard of 3 x 3-pixel
    squares (sharp edges, where the cubic overshoots)."""
    if image == "checker":
        y, x = np.mgrid[:h, :w]
        sq = np.where((y // 3 + x // 3) % 2 == 0, 0, 255).astype(np.uint8)
        return np.ascontiguousarray(np.broadcast_to(sq[:, :, None], (h, w, c)))
    return P.case_image(h, w, c, image, seed)


# The cases only the bicubic fixture holds, after the 32 of pil_resize_oracle.GOLDEN_CASES: a 0 / 255 checkerboard
# upscaled about 5x, whose sums leave [0, 255 * 2^22] in both passes, and a 1 x 16384 image stretched to 224 x 224 --
# the most taps the Net's 16384-pixel limit allows (292 non-zero of kmax 295).
OVERSHOOT_CASE = (45, 40, 3, 0, 224, 200, "checker")
LONGEST_CASE = (1, 16384, 3, 0, 224, 224, "random")
# (h, w, c, resize_short, out_h, out_w, image) of tests/golden/pil_bicubic_resize.json (tools/make_pil_resize_golden.py);
# case i uses seed i
GOLDEN_CASES = list(P.GOLDEN_CASES) + [OVERSHOOT_CASE, LONGEST_CASE]
