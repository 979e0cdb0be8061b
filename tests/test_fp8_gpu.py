"""GPU: the E4M3 conv kind bit for bit against the numpy restatement (tests/fp8_oracle.py).

1. The accumulator probe: one 32-byte k slice with one large product and one small one, 2^16 + 2^(16 - t), for every
   shift t the operands reach. It reports the widest shift the tensor cores keep and asserts it covers the designed
   data's bound (fp8_oracle.EXACT_BITS); a second probe reports what happens to 3/4 of the first unit it drops.
2. Designed data whose every partial sum is exact within that width: the im2col kernel at every tile width, split-K
   2 / 4 / 8 (twice, identical bits), the slab kernel, its fused MAX pooling and the persistent kernel, with e4m3 and
   fp32 outputs, e4m3 residuals and relu. Padding channels past the 16-byte unit of channel k - 1 keep a sentinel; the
   channels of that unit past k come back as +0, as the int8 kind's do (test_8bit_store_writes_the_last_16_byte_unit_whole).
"""
import numpy as np
import pytest

import fp8_oracle as E
import float_exact as F
from anakin_b200 import saber_abi as A
from test_conv_gpu import PERSISTENT_CASES, POOL_CASES, SLAB_CASES, SPLIT_CASES
from test_float_exact_gpu import use_kernel

pytestmark = pytest.mark.gpu

SENTINEL_CODE = 0x5A


def run_e4m3(x, w, bias, scale, out_fp32, res=None, sum_scale=1.0, relu=False, stride=(1, 1), pad=(0, 0),
             dil=(1, 1), **kw):
    """One E4M3 plan into a sentinel-filled output whose row pitch exceeds k: (output [..., :k], plan info)."""
    import torch
    from gpu_util import ConvRunner, dev, pad_channels
    k = w.shape[0]
    out_dt = A.FLOAT if out_fp32 else A.FP8E4M3
    ldc = F.ldc_for(k, A.FLOAT if out_fp32 else A.UINT8, A.UINT8 if res is not None else None)
    run = ConvRunner(A.MATH_E4M3, x.shape, A.FP8E4M3, w, bias, scale, out_dt,
                     res_dtype=A.FP8E4M3 if res is not None else -1, sum_scale=sum_scale, ldc=ldc, stride=stride,
                     pad=pad, dil=dil, relu=relu, **kw)
    info = run.info()
    shape = (x.shape[0], run.ho, run.wo, ldc)
    if out_fp32:
        out = torch.full(shape, -777.0, dtype=torch.float32, device="cuda")
    else:
        out = torch.full(shape, SENTINEL_CODE, dtype=torch.uint8, device="cuda")
    run.run(dev(x), dev(pad_channels(res, ldc)) if res is not None else None, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    if out_fp32:
        pad_ok = (got[..., k:] == -777.0).all()
    else:
        # The TMA tile store writes the 16-byte unit that holds channel k - 1 whole, as for the int8 kind's 8-bit
        # outputs (test_8bit_store_writes_the_last_16_byte_unit_whole): its channels past k carry the staged values of
        # channels with zero weights, bias 0 and a zero residual, +0 codes. Every later channel keeps the sentinel.
        k16 = (k + 15) // 16 * 16
        pad_ok = (got[..., k:k16] == 0).all() and (got[..., k16:] == SENTINEL_CODE).all()
    assert pad_ok, "padding channels past k must keep the sentinel (info %s)" % info
    return got[..., :k], info


def assert_codes(got, want, info=None):
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    view = np.uint32 if got.dtype == np.float32 else np.uint8
    bad = np.argwhere(got.view(view) != want.view(view))
    assert bad.shape[0] == 0, "%d of %d differ, first %s: got %s want %s (info %s)" % (
        bad.shape[0], got.size, bad[:5].tolist(), got[tuple(bad[:5].T)], want[tuple(bad[:5].T)], info)


# name: (fp32 output, e4m3 residual, relu)
VARIANTS = {"e": (False, False, False), "e_res_relu": (False, True, True), "e_relu": (False, False, True),
            "f": (True, False, False), "f_res": (True, True, False)}


def designed_run(geom, variant, **kw):
    out_fp32, with_res, relu = VARIANTS[variant]
    n, h, w, c, k, r, s, stride, ph, pw, dil = geom
    x, wc, bias, scale, res, ss, want = E.designed_case(geom, out_fp32, with_res, relu, variant)
    got, info = run_e4m3(x, wc, bias, scale, out_fp32, res, ss, relu, stride=(stride, stride), pad=(ph, pw),
                         dil=(dil, dil), **kw)
    return got, want, info


# ================================================================================ 1. accumulator probe
def test_accumulator_probe():
    """Row (a, b) of a 1x1 conv over 32 channels: x = [256, 2^a, 0...], output channel j: w = [256, 2^b_j, 0...], so
    the exact sum is 2^16 + 2^(a + b_j). fp32 output, bias 0, scale 1: the stored value is the accumulator. The shift
    t = 16 - (a + b) the tensor cores still add exactly is the accumulator's width below the largest product."""
    rows = [8, 0, -9]                                      # a
    bs = list(range(-9, 9))                                # b_j (E4M3 exponents -9..8)
    c, k = 32, 32
    x = np.zeros((1, 1, len(rows), c), np.float32)
    x[0, 0, :, 0] = 256
    x[0, 0, :, 1] = [2.0 ** a for a in rows]
    w = np.zeros((k, c, 1, 1), np.float32)
    w[:, 0] = 256
    w[:len(bs), 1, 0, 0] = [2.0 ** b for b in bs]
    w[len(bs):, 1, 0, 0] = 0
    got, info = run_e4m3(E.encode(x), E.encode(w), np.zeros(k, np.float32), np.ones(k, np.float32), True)
    kept = {}
    for i, a in enumerate(rows):
        for j, b in enumerate(bs):
            t = 16 - (a + b)
            exact = 2.0 ** 16 + 2.0 ** (a + b)
            if float(np.float32(exact)) != exact:
                continue                                    # not an fp32 number: beyond what the store can show
            kept.setdefault(t, []).append(float(got[0, 0, i, j]) == exact)
    shifts = sorted(kept)
    width = 0
    for t in shifts:
        if not all(kept[t]):
            break
        width = t
    print("e4m3 accumulator probe: exact up to a shift of %d bits below the largest product (shifts %d..%d tried); "
          "per shift: %s" % (width, shifts[0], shifts[-1], {t: all(kept[t]) for t in shifts}))
    assert width >= E.EXACT_BITS, "the designed data need %d bits, the accumulator keeps %d" % (E.EXACT_BITS, width)


def test_accumulator_probe_rounding():
    """Information, not a gate: 2^16 + 2^(16 - w - 1) + 2^(16 - w - 2) for the probe's width w = 13 (so 3/4 of the
    first dropped unit): round to nearest gives 2^16 + 2^(16 - w), dropping the bits gives 2^16. Three products of one
    k slice, fp32 output, bias 0, scale 1, in both orders of the small products."""
    c, k, w_bits = 32, 32, 13
    small = [2.0 ** (16 - w_bits - 1), 2.0 ** (16 - w_bits - 2)]
    x = np.zeros((1, 1, 2, c), np.float32)
    x[0, 0, 0, :3] = [256, small[0], small[1]]
    x[0, 0, 1, :3] = [256, small[1], small[0]]
    w = np.zeros((k, c, 1, 1), np.float32)
    w[0, :3, 0, 0] = 256, 1, 1
    got, _ = run_e4m3(E.encode(x), E.encode(w), np.zeros(k, np.float32), np.ones(k, np.float32), True)
    ulp = 2.0 ** (16 - w_bits)
    for row in range(2):
        v = float(got[0, 0, row, 0]) - 2.0 ** 16
        mode = {0.0: "dropped", ulp: "rounded to nearest", 0.75 * ulp: "kept"}.get(v, "other")
        print("e4m3 accumulator rounding probe: 2^16 + 3/4 ulp (order %d) -> 2^16 %+g: %s" % (row, v, mode))


# ================================================================================ 2. designed data, every conv path
IM2COL_CASES = [
    (1, 12, 12, 32, 32, 3, 3, 1, 1, 1, 1),
    (3, 21, 21, 16, 24, 3, 3, 2, 1, 1, 1),
    (2, 24, 24, 64, 64, 1, 1, 1, 0, 0, 1),
    (1, 36, 36, 32, 48, 3, 3, 1, 2, 2, 2),
    (2, 28, 28, 128, 128, 3, 3, 1, 1, 1, 1),
    (1, 56, 56, 64, 64, 1, 1, 2, 0, 0, 1),
    (1, 14, 14, 256, 200, 3, 3, 1, 1, 1, 1),
]
WIDTHS = [32, 64, 128, 256]
VN = list(VARIANTS)


@pytest.mark.parametrize("variant", VN)
@pytest.mark.parametrize("case", IM2COL_CASES)
def test_designed_im2col(case, variant, monkeypatch):
    bn = WIDTHS[(IM2COL_CASES.index(case) + VN.index(variant)) % 4]
    bn = min(bn, 128 if VARIANTS[variant][0] else 256)
    use_kernel(monkeypatch, "im2col", bn=bn)
    got, want, info = designed_run(case, variant)
    assert info["block_n"] == bn and not info["slab"] and not info["persistent"], info
    assert_codes(got, want, info)


@pytest.mark.parametrize("variant", ["e_res_relu", "f"])
@pytest.mark.parametrize("case,bn,split", SPLIT_CASES)
def test_designed_split_k(case, bn, split, variant, monkeypatch):
    """fp32 partial sums in rank order: exact here, and identical bits on a second run."""
    use_kernel(monkeypatch, "im2col", bn=bn, split=split)
    geom = F.full_geom(case)
    got, want, info = designed_run(geom, variant)
    assert (info["block_n"], info["split"]) == (bn, split) and not info["slab"], info
    assert_codes(got, want, info)
    again, _, _ = designed_run(geom, variant)
    assert_codes(again, got, info)


@pytest.mark.parametrize("variant", ["e_res_relu", "e", "f"])
@pytest.mark.parametrize("case", SLAB_CASES)
def test_designed_slab(case, variant, monkeypatch):
    n, h, w, c, k, r, s, ph, pw = case
    bn = min([0, 32, 64, 128, 256][(SLAB_CASES.index(case) + VN.index(variant)) % 5],
             128 if VARIANTS[variant][0] else 256, 64 if max(r, s) > 3 else 256)
    use_kernel(monkeypatch, "slab", bn=bn)
    got, want, info = designed_run((n, h, w, c, k, r, s, 1, ph, pw, 1), variant)
    assert info["slab"] and (not bn or info["block_n"] == bn), info
    assert_codes(got, want, info)


@pytest.mark.parametrize("variant", ["e_res_relu", "f_res"])
@pytest.mark.parametrize("case", PERSISTENT_CASES)
def test_designed_persistent(case, variant, monkeypatch):
    n, h, w, c, k, r, stride, pad = case
    use_kernel(monkeypatch, "persistent", bn=128 if k >= 128 else 0)
    got, want, info = designed_run((n, h, w, c, k, r, r, stride, pad, pad, 1), variant)
    assert info["persistent"] and not info["slab"], info
    assert_codes(got, want, info)


@pytest.mark.parametrize("variant", ["e", "e_relu", "f"])
@pytest.mark.parametrize("case", [POOL_CASES[0], POOL_CASES[3], POOL_CASES[4], POOL_CASES[5]])
def test_designed_fused_max_pool(case, variant, monkeypatch):
    """The slab kernel's fused MAX pooling: e4m3 outputs compare decoded values and keep the codes (-0 and +0 tie, the
    first one visited stays); fp32 outputs of the e4m3 kind pool as floats."""
    n, h, w, c, k, r, pad, pk, ps, pp = case
    geom = (n, h, w, c, k, r, r, 1, pad, pad, 1)
    out_fp32, with_res, relu = VARIANTS[variant]
    x, wc, bias, scale, _, _, conv = E.designed_case(geom, out_fp32, False, relu, variant)
    pd = A.PoolDesc(dtype=A.FLOAT if out_fp32 else A.FP8E4M3, type=A.POOL_MAX, n=n, h=conv.shape[1], w=conv.shape[2], c=k, window_h=pk,
                    window_w=pk, pad_h=pp, pad_w=pp, stride_h=ps, stride_w=ps)
    import ctypes as C
    ho, wo = C.c_int32(), C.c_int32()
    A.check(A.load().b200_pool_out_hw(C.byref(pd), C.byref(ho), C.byref(wo)), "pool_out_hw")
    want = E.max_pool(conv, pk, ps, pp, (ho.value, wo.value), codes=not out_fp32)
    if out_fp32:   # the data must tell a float pooling from a bytewise one: most pooled values have mixed-sign windows
        assert (want != 0).mean() > 0.5 and (conv < 0).any()
    got, info = run_e4m3(x, wc, bias, scale, out_fp32, relu=relu, pad=(pad, pad), fuse_pool=pk, pool_stride=ps,
                         pool_pad=pp)
    assert info["slab"], info
    assert_codes(got, want, info)


@pytest.mark.parametrize("kernel", ["im2col", "slab"])
@pytest.mark.parametrize("k", [24, 40, 200])
def test_8bit_store_writes_the_last_16_byte_unit_whole(k, kernel, monkeypatch):
    """The int8 and e4m3 kinds store their 8-bit outputs through the same TMA tile maps (inner extent k). When k is not
    a multiple of 16, both write the channels past k of the 16-byte unit that holds channel k - 1 -- with the staged
    values of the channels past k, 0 -- and nothing after it. This pins that the e4m3 kind behaves as the int8 kind."""
    import torch
    from gpu_util import ConvRunner, dev
    use_kernel(monkeypatch, kernel)
    c, ldc, k16 = 32, (k + 15) // 16 * 16 + 16, (k + 15) // 16 * 16
    x = np.full((1, 12, 12, c), 0x38, np.uint8)          # e4m3 1.0, u8 56
    w = np.full((k, c, 3, 3), 0x01, np.uint8)            # e4m3 2^-9, s8 1
    for math, din in ((A.MATH_I8, A.UINT8), (A.MATH_E4M3, A.FP8E4M3)):
        run = ConvRunner(math, x.shape, din, w, np.full(k, 3.0, np.float32), np.full(k, 0.001, np.float32),
                         din, pad=(1, 1), ldc=ldc)
        out = torch.full((1, run.ho, run.wo, ldc), SENTINEL_CODE, dtype=torch.uint8, device="cuda")
        run.run(dev(x), None, out)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert run.info()["slab"] == (kernel == "slab"), run.info()
        assert (got[..., :k] != SENTINEL_CODE).all() and (got[..., k:k16] == 0).all(), (math, kernel)
        assert (got[..., k16:] == SENTINEL_CODE).all(), (math, kernel)


def test_e4m3_plan_refuses_int8_edges():
    from gpu_util import ConvRunner
    x = np.zeros((1, 8, 8, 32), np.uint8)
    w = np.zeros((32, 32, 3, 3), np.uint8)
    with pytest.raises(A.SaberError, match="SaberInvalidValue"):
        ConvRunner(A.MATH_E4M3, x.shape, A.UINT8, w, None, None, A.FP8E4M3, pad=(1, 1))
    with pytest.raises(A.SaberError, match="SaberInvalidValue"):
        ConvRunner(A.MATH_E4M3, x.shape, A.FP8E4M3, w, None, None, A.UINT8, pad=(1, 1))
