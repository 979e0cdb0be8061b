"""CPU suite for the E4M3 conv kind: the numpy codec against torch.float8_e4m3fn, the oracle's exactness bound, the
designed data's bound, the planner (E4M3 plans as INT8 at every ResNet-50 shape) and the one place the encoder lives."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest

import fp8_oracle as E
from test_cpu_conv_plan import H100_SXM_SMS, set_switches

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "anakin_b200", "csrc")


def _torch_encode(x):
    torch = pytest.importorskip("torch")
    t = torch.from_numpy(np.clip(np.asarray(x, np.float32), -448, 448))
    return t.to(torch.float8_e4m3fn).view(torch.uint8).numpy()


# ------------------------------------------------------------------------------------------------ codec
def test_decode_matches_torch_on_all_codes():
    torch = pytest.importorskip("torch")
    codes = np.arange(256, dtype=np.uint8)
    want = torch.from_numpy(codes).view(torch.float8_e4m3fn).float().numpy().astype(np.float64)
    got = E.decode(codes)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.isnan(got).sum() == 2
    ok = ~np.isnan(got)
    assert np.array_equal(got[ok], want[ok]) and np.array_equal(np.signbit(got[ok]), np.signbit(want[ok]))
    assert E.decode(0x7E) == 448 and E.decode(0x01) == 2.0 ** -9


def test_encode_round_trips_every_finite_code():
    codes = np.array([c for c in range(256) if c not in (0x7F, 0xFF)], np.uint8)
    assert np.array_equal(E.encode(E.decode(codes).astype(np.float32)), codes)
    assert np.array_equal(_torch_encode(E.decode(codes)), codes)


def test_encode_ties_round_to_even_as_torch():
    v = E.decode(np.arange(127, dtype=np.uint8))
    mids = ((v[:-1] + v[1:]) / 2).astype(np.float32)              # exact in fp32: every midpoint of the grid
    assert (mids.astype(np.float64) == (v[:-1] + v[1:]) / 2).all()
    for sign in (1, -1):
        x = sign * mids
        got = E.encode(x)
        assert np.array_equal(got, _torch_encode(x))
        assert ((got & 1) == 0).all(), "a tie must land on the even code"
        # one fp32 ulp either side of every tie
        for d in (np.inf, -np.inf):
            y = np.nextafter(x, np.float32(d))
            assert np.array_equal(E.encode(y), _torch_encode(y))


def test_encode_saturates_and_matches_torch_on_random_values():
    rng = np.random.default_rng(8)
    x = np.concatenate([rng.standard_normal(200000) * 10.0 ** rng.uniform(-4, 3, 200000),
                        [448, 449, 463.99, 464, 465, 480, 1e30, -1e30, 2.0 ** -10, -2.0 ** -10, 2.0 ** -10 * 1.0001,
                         0.0, -0.0]]).astype(np.float32)
    got = E.encode(x)
    assert np.array_equal(got, _torch_encode(x))
    big = np.abs(x) >= 448
    assert (got[big] & 0x7F == 0x7E).all(), "beyond the range the encoder saturates to +-448"
    assert E.encode(np.float32(-0.0)) == 0x80 and E.encode(np.float32(-2.0 ** -11)) == 0x80
    assert E.encode(np.float32(np.nan)) == 0x7F


# ------------------------------------------------------------------------------------------------ oracle bounds
def test_oracle_sum_is_exact_and_asserts_its_bound():
    x = np.full((1, 1, 1, 64), 0x7E, np.uint8)                    # 448
    w = np.full((2, 64, 1, 1), 0x7E, np.uint8)
    w[1] = 0x01                                                    # 2^-9
    acc = E.conv(x, w)
    assert acc[0, 0, 0, 0] == 64 * 448.0 ** 2 and acc[0, 0, 0, 1] == 64 * 448 * 2.0 ** -9
    # 448^2 is 2^35.6 units of 2^-18: 2^17 such products stay below 2^53 units, 2^18 do not
    big = np.full((1, 1, 1, 1 << 17), 0x7E, np.uint8)
    assert E.conv(big, np.full((1, 1 << 17, 1, 1), 0x7E, np.uint8))[0, 0, 0, 0] == (1 << 17) * 448.0 ** 2
    with pytest.raises(AssertionError, match="not exact"):
        E.conv(np.full((1, 2, 2, 1 << 16), 0x7E, np.uint8), np.full((1, 1 << 16, 2, 2), 0x7E, np.uint8))


def test_epilogue_restatement():
    acc = np.array([[3.0, -5.0, 100.0, 0.0]])
    bias = np.array([0.5, 0.0, 1e6, -1.0], np.float32)
    scale = np.array([1.0, 2.0, 1.0, 2.0 ** -12], np.float32)
    codes = E.epilogue(acc, bias, scale)
    assert E.decode(codes)[0, 0] == 3.5 and E.decode(codes)[0, 1] == -10 and E.decode(codes)[0, 2] == 448
    assert codes[0, 3] == 0x80                                    # -2^-12 rounds to -0
    assert E.epilogue(acc, bias, scale, relu=True)[0, 3] == 0x00  # relu gives +0
    f = E.epilogue(acc, bias, scale, out_fp32=True)
    assert f.dtype == np.float32 and f[0, 2] == np.float32(1e6 + 100)


@pytest.mark.parametrize("geom", [(1, 7, 7, 512, 64, 3, 3, 1, 1, 1, 1), (2, 9, 9, 2048, 32, 1, 1, 1, 0, 0, 1),
                                  (1, 12, 12, 32, 48, 3, 3, 1, 1, 1, 1)])
def test_designed_data_stay_within_the_exact_bound(geom):
    x, w, bias, scale, res, ss, want = E.designed_case(geom, False, True, True, "cpu")
    acc = E.conv(x, w, stride=(geom[7],) * 2, pad=(geom[8], geom[9]), dil=(geom[10],) * 2)
    units = E.F.conv_f64(np.abs(E.decode(x)), np.abs(E.decode(w)), (geom[7],) * 2, (geom[8], geom[9]),
                         (geom[10],) * 2) / 2.0 ** (E.X_EXP + E.W_EXP)
    assert units.max() <= 2 ** E.EXACT_BITS and units.max() > 2 ** (E.EXACT_BITS - 2)
    # the store's rounding is reached: most nonzero values are not the fp32 value before it
    f = E.epilogue(acc, bias, scale, res, ss, True, out_fp32=True)
    assert (E.decode(want) != f)[f != 0].mean() > 0.5
    assert ((want & 0x7F) == 0x7E).any(), "no saturated output"


# ------------------------------------------------------------------------------------------------ planner
def _resnet50_convs():
    """(h, c, k, r, stride, pad, with_res) of every ResNet-50 conv the conv plan runs (the 7x7 stem aside), at the
    input size of each layer, and the classifier as a 1x1 conv."""
    out = []
    h, c = 56, 64
    for stage, (mid, width, blocks) in enumerate([(64, 256, 3), (128, 512, 4), (256, 1024, 6), (512, 2048, 3)]):
        for b in range(blocks):
            stride = 2 if (b == 0 and stage > 0) else 1
            if b == 0:
                out.append((h, c, width, 1, stride, 0, False))                # branch1
            out.append((h, c, mid, 1, stride, 0, False))                      # branch2a
            h2 = h // stride
            out.append((h2, mid, mid, 3, 1, 1, False))                        # branch2b
            out.append((h2, mid, width, 1, 1, 0, True))                       # branch2c + residual
            h, c = h2, width
    return out


def _desc(math, n, layer, fp32_out=False):
    from anakin_b200 import saber_abi as A
    h, c, k, r, stride, pad, with_res = layer
    if math == A.MATH_I8:
        din, dout, dres = A.UINT8, A.FLOAT if fp32_out else A.UINT8, A.INT8
    else:
        din, dout, dres = A.FP8E4M3, A.FLOAT if fp32_out else A.FP8E4M3, A.FP8E4M3
    return A.ConvDesc(math=math, in_dtype=din, out_dtype=dout, res_dtype=dres if with_res else -1, n=n, h=h, w=h, c=c,
                      k=k, ldc=k, r=r, s=r, pad_h=pad, pad_w=pad, stride_h=stride, stride_w=stride, dil_h=1, dil_w=1,
                      relu=1, sum_scale=1.0)


def _choice(desc):
    from anakin_b200 import saber_abi as A
    out = A.ConvPlanChoice()
    st = A.load().b200_conv_plan_choose(C.byref(desc), H100_SXM_SMS, C.byref(out))
    return st, tuple(getattr(out, f) for f, _ in A.ConvPlanChoice._fields_)


@pytest.mark.parametrize("n", [1, 8, 32])
def test_e4m3_plans_are_the_int8_plans_at_every_resnet50_shape(n, monkeypatch):
    from anakin_b200 import saber_abi as A
    set_switches(monkeypatch, {})
    layers = _resnet50_convs() + [(1, 2048, 1000, 1, 1, 0, False)]
    kinds = set()
    for i, layer in enumerate(layers):
        fp32_out = i == len(layers) - 1
        st8, c8 = _choice(_desc(A.MATH_I8, n, layer, fp32_out))
        ste, ce = _choice(_desc(A.MATH_E4M3, n, layer, fp32_out))
        assert st8 == A.SUCCESS and (ste, ce) == (st8, c8), (n, layer, c8, ce)
        kinds.add((c8[0], c8[2] > 1))
    assert {k for k, _ in kinds} >= {A.CONV_KERNEL_TILE, A.CONV_KERNEL_SLAB}


def test_e4m3_plans_refuse_other_dtypes(monkeypatch):
    from anakin_b200 import saber_abi as A
    set_switches(monkeypatch, {})
    layer = (14, 256, 256, 3, 1, 1, True)
    assert _choice(_desc(A.MATH_E4M3, 8, layer))[0] == A.SUCCESS
    for field, dt in [("in_dtype", A.UINT8), ("in_dtype", A.FLOAT), ("out_dtype", A.HALF), ("out_dtype", A.INT8),
                      ("res_dtype", A.INT8), ("res_dtype", A.FLOAT)]:
        d = _desc(A.MATH_E4M3, 8, layer)
        setattr(d, field, dt)
        assert _choice(d)[0] == A.INVALID_VALUE, (field, dt)
    # and the other kinds refuse e4m3 edges
    for math, din in [(A.MATH_I8, A.UINT8), (A.MATH_F16, A.HALF), (A.MATH_TF32X3, A.FLOAT)]:
        d = _desc(A.MATH_E4M3, 8, layer)
        d.math, d.in_dtype, d.out_dtype, d.res_dtype = math, din, A.FP8E4M3, -1
        assert _choice(d)[0] == A.INVALID_VALUE, math


# ------------------------------------------------------------------------------------------------ sources
def test_e4m3_encoder_lives_in_the_codec():
    found = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "**", "*"), recursive=True)):
        if path.endswith((".cu", ".cuh", ".h", ".cpp")):
            with open(path) as f:
                code = re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S))
            for token in ("cvt.rn.satfinite.e4m3x2", "cvt.rn.f16x2.e4m3x2"):
                if token in code:
                    found.setdefault(token, set()).add(os.path.relpath(path, CSRC))
    assert found == {"cvt.rn.satfinite.e4m3x2": {"vec.cuh"}, "cvt.rn.f16x2.e4m3x2": {"vec.cuh"}}
