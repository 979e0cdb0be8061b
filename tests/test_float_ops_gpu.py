"""The float kernels between the convolutions of FP32 and FP16 nets, on designed data, against tests/float_ops_ref.py:
eltwise, activation and scale bit for bit against op-for-op restatements (f16 and f32); sigmoid, tanh, ELU and softmax
against float64 within bounds derived from CUDA's documented expf / tanhf errors; the float SE gate bit for bit
against the restatement of its pooling order, and within a derived bound of the float64 gate."""
import ctypes as C

import numpy as np
import pytest

import float_ops_ref as R
import se_oracle as S

pytestmark = pytest.mark.gpu

F32, F16 = np.float32, np.float16


def _lib():
    from anakin_b200 import saber_abi as A
    return A, A.load()


def _grid_threads():
    """Threads of the pointwise kernels' largest grid: 16 CTAs of 256 per SM (grid_for in pointwise.cu)."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256


def _dt(np_dt):
    from anakin_b200 import saber_abi as A
    return A.HALF if np_dt == F16 else A.FLOAT


# ------------------------------------------------------------------------------------------------ eltwise
def _eltwise(a, b, op, c0, c1, relu):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    A, lib = _lib()
    ad, bd = dev(a), dev(b)
    out = torch.empty_like(ad)
    dt = _dt(a.dtype)
    A.check(lib.b200_eltwise_run(dt, dt, dt, op, ptr(ad), ptr(bd), ptr(out), a.size, c0, c1, int(relu), stream_ptr()),
            "eltwise")
    torch.cuda.synchronize()
    return out.cpu().numpy()


# 1: a tail only; 7: one float4 and a tail of 3; 8: two float4s, no tail; 100003: odd tail; 2500003: several
# grid-stride passes of both kernels (asserted against the device's grid)
ELT_COUNTS = [1, 7, 8, 100003, 2500003]


@pytest.mark.parametrize("count", ELT_COUNTS)
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("op", [R.ELT_PROD, R.ELT_SUM, R.ELT_MAX])
@pytest.mark.parametrize("dt", [F16, F32], ids=["f16", "f32"])
def test_eltwise_bit_exact(dt, op, relu, count):
    a, b = R.eltwise_data(dt, count)
    if count > 2000000:
        assert count // (4 if dt == F32 else 1) > _grid_threads()
    got = _eltwise(a, b, op, 1.0, 1.0, relu)
    R.assert_same_bits(got, R.eltwise(a, b, op, 1.0, 1.0, relu), "op %d relu %d" % (op, relu))
    if relu and count >= 100:
        # the designed -0 results come out as +0 (PTX max.f32 orders -0 below +0)
        pre = R.eltwise(a, b, op, 1.0, 1.0, False)
        neg0 = (pre == 0) & np.signbit(pre)
        assert neg0.any() and not np.signbit(got[neg0]).any()


@pytest.mark.parametrize("dt", [F16, F32], ids=["f16", "f32"])
def test_eltwise_sum_coefficients(dt):
    """SUM rounds c0 * a and c1 * b on their own before the add (no FMA)."""
    a, b = R.eltwise_data(dt, 100003)
    for relu in (False, True):
        got = _eltwise(a, b, R.ELT_SUM, 0.7, -1.3, relu)
        R.assert_same_bits(got, R.eltwise(a, b, R.ELT_SUM, 0.7, -1.3, relu), "sum 0.7 / -1.3")


# ------------------------------------------------------------------------------------------------ activation
def _activation(x, act, slope=0.0, coef=1.0):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    A, lib = _lib()
    xd = dev(x)
    out = torch.empty_like(xd)
    A.check(lib.b200_activation_run(_dt(x.dtype), act, ptr(xd), ptr(out), x.size, slope, coef, stream_ptr()),
            "activation")
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("act,slope,coef", [(R.ACT_RELU, 0.0, 0.0), (R.ACT_RELU, 0.1, 0.0),
                                            (R.ACT_CLIPPED_RELU, 0.0, 6.0)], ids=["relu", "leaky0.1", "relu6"])
def test_activation_f16_relu_kinds_all_codes(act, slope, coef):
    x = R.all_f16_codes()
    got = _activation(x, act, slope, coef)
    R.assert_same_bits(got, R.relu_kinds(x, act, slope, coef))


@pytest.mark.parametrize("act", [R.ACT_SIGMOID, R.ACT_TANH, R.ACT_ELU], ids=["sigmoid", "tanh", "elu"])
def test_activation_f16_transcendental_all_codes(act):
    """Every f16 code: the correctly rounded f16 of the float64 value, except where the fp32 intermediate lies within
    its derived bound of an f16 rounding boundary; there the result must still lie between the f16 roundings of the
    bound's ends (R.check_act_f16). Where that interval holds just two f16 numbers, at most 1% of the codes may take
    the other one. Where it holds more -- ELU for small negative x, whose expf(x) - 1 cancels -- the interval is the
    check."""
    x = R.all_f16_codes()
    got = _activation(x, act, 0.0, 1.0)
    bad, near, wide, off = R.check_act_f16(got, x, act, 1.0)
    assert not bad.any(), (int(bad.sum()), x[bad][:8].tolist(), got[bad][:8].tolist())
    ulps = np.abs(R.f16_ordinal(got) - R.f16_ordinal(R.act_f64(x, act, 1.0).astype(F16)))[off]
    print("f16 act %d: %d codes near a rounding boundary (%d with more than one ulp of doubt); %d differ from the "
          "correctly rounded f16 by 1 ulp, %d by more (at most %d)" % (act, int(near.sum()), int(wide.sum()),
                                                                     int((ulps == 1).sum()), int((ulps > 1).sum()),
                                                                     int(ulps.max()) if ulps.size else 0))
    assert (off & ~wide).sum() <= 655
    if act != R.ACT_ELU:
        assert not wide.any()


@pytest.mark.parametrize("act,slope,coef", [(R.ACT_RELU, 0.0, 0.0), (R.ACT_RELU, 0.1, 0.0),
                                            (R.ACT_CLIPPED_RELU, 0.0, 6.0)], ids=["relu", "leaky0.1", "relu6"])
def test_activation_f32_relu_kinds(act, slope, coef):
    x = R.f32_activation_grid()
    got = _activation(x, act, slope, coef)
    R.assert_same_bits(got, R.relu_kinds(x, act, slope, coef))


@pytest.mark.parametrize("act,coef", [(R.ACT_SIGMOID, 1.0), (R.ACT_TANH, 1.0), (R.ACT_ELU, 1.5)],
                         ids=["sigmoid", "tanh", "elu"])
def test_activation_f32_transcendental_bounds(act, coef):
    x = R.f32_activation_grid()
    got = _activation(x, act, 0.0, coef)
    ratio, bad = R.check_act_f32(got, x, act, coef)
    assert not bad.any(), (ratio, x[bad][:8].tolist(), got[bad][:8].tolist())
    if act == R.ACT_ELU:
        pos = x > 0
        R.assert_same_bits(got[pos], x[pos], "ELU is the identity above 0")


# ------------------------------------------------------------------------------------------------ scale
# (pixels, channels, stored channels): 3 / 24 / 1000 channels, a padded channel_stored, and 4096 x 1000 elements, several
# grid-stride passes of the capped grid
SCALE_CASES = [(777, 3, 3), (301, 24, 24), (64, 1000, 1000), (33, 1000, 1008), (4096, 1000, 1000)]


@pytest.mark.parametrize("case", SCALE_CASES, ids=lambda c: "%dx%d_%d" % c)
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("dt", [F16, F32], ids=["f16", "f32"])
def test_scale_bit_exact(dt, bias, case):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    A, lib = _lib()
    pixels, c, cs = case
    x, w, b = R.scale_data(dt, pixels, c, cs)
    if pixels * cs > 4000000:
        assert pixels * cs > 4 * _grid_threads()
    xd, wd, bd = dev(x), dev(w), dev(b)
    out = torch.empty_like(xd)
    A.check(lib.b200_scale_run(_dt(dt), ptr(xd), ptr(out), pixels, cs, ptr(wd), ptr(bd) if bias else None,
                               stream_ptr()), "scale")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    R.assert_same_bits(got, R.scale(x, w, b if bias else None))


# ------------------------------------------------------------------------------------------------ softmax
def _softmax(x, outer, length, inner):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    A, lib = _lib()
    xd = dev(x)
    out = torch.empty_like(xd)
    A.check(lib.b200_softmax_run(ptr(xd), ptr(out), outer, length, inner, stream_ptr()), "softmax")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def test_softmax_exact_rows():
    for x, want in R.softmax_exact_rows():
        got = _softmax(x[None], 1, x.size, 1)[0]
        R.assert_same_bits(got, want, "len %d" % x.size)


def test_softmax_strided_exact():
    """Equal logits along a non-innermost axis of 64: each column sums 64 exact ones, so every output is 1/64."""
    x = np.full((2, 64, 70), -7.5, F32)
    got = _softmax(x, 2, 64, 70)
    R.assert_same_bits(got, np.full(x.shape, 1 / 64, F32))


@pytest.mark.parametrize("length", R.SOFTMAX_LENGTHS)
def test_softmax_rows_bounded(length):
    x = R.softmax_bounded_rows(length)
    got = _softmax(x, x.shape[0], length, 1)
    err = np.abs(got.astype(np.float64) - R.softmax_f64(x))
    bound = R.softmax_bound(x, R.rows_adds(length))
    assert (err <= bound).all(), float((err / bound).max())
    assert got[0, 1] == 0 and not np.signbit(got[0, 1])        # the -inf logit


def test_softmax_pitched_rows():
    """b200_softmax_rows over pitched rows: NaN in the input's gap must not reach the row, and the output's gap keeps
    its sentinel."""
    import torch
    from gpu_util import dev, ptr, stream_ptr
    A, lib = _lib()
    rows, length, ip, op = 5, 1000, 1031, 1040
    x = np.full((rows, ip), np.nan, F32)
    x[:, :length] = np.concatenate([R.softmax_bounded_rows(length), R.softmax_bounded_rows(length)[:2]])
    sentinel = np.float32(-12345.678)
    xd = dev(x)
    out = torch.full((rows, op), float(sentinel), dtype=torch.float32, device="cuda")
    A.check(lib.b200_softmax_rows(ptr(xd), ptr(out), rows, length, ip, op, stream_ptr()), "softmax_rows")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    R.assert_same_bits(got[:, length:], np.full((rows, op - length), sentinel, F32), "output gap")
    v = x[:, :length]
    err = np.abs(got[:, :length].astype(np.float64) - R.softmax_f64(v))
    assert (err <= R.softmax_bound(v, R.rows_adds(length))).all()


# (outer, axis, inner): outer * inner above one 128-thread block
@pytest.mark.parametrize("shape", [(3, 21, 77), (2, 1000, 300), (5, 257, 31)], ids=lambda s: "%dx%dx%d" % s)
def test_softmax_strided_bounded(shape):
    outer, length, inner = shape
    assert outer * inner > 128
    rows = R.softmax_bounded_rows(length)
    x = np.stack([rows[i % 3] for i in range(outer * inner)]).reshape(outer, inner, length)
    x = np.ascontiguousarray(np.transpose(x, (0, 2, 1)))
    got = _softmax(x, outer, length, inner)
    err = np.abs(got.astype(np.float64) - R.softmax_f64(x, axis=1))
    assert (err <= R.softmax_bound(x, length, axis=1)).all()


# ------------------------------------------------------------------------------------------------ SE gate
# (dtype, n, hw, c, ld, r, ldg, W2 at an address that is not 16-byte aligned)
SE_CASES = [
    (F32, 2, 49, 2048, 2048, 128, 2048, False),   # 512 vectors per pixel: one slot, every rank pools 7 pixels
    (F32, 3, 7, 64, 72, 16, 80, False),           # ld > c (NaN in the padding), 14 slots; hw 7: rank 7 pools nothing
    (F16, 17, 1, 96, 104, 6, 100, True),          # hw 1: ranks 1-7 pool nothing; 17 images loop; r % 4: scalar W2
    (F16, 4, 3136, 256, 256, 16, 264, True),      # 8 slots of 49 pixels per rank; r % 4 == 0 but W2 unaligned: scalar
    (F32, 20, 49, 512, 512, 32, 520, False),      # 2 slots; 20 images over 16 clusters; the float4 W2 path
    (F16, 2, 9, 2048, 2048, 128, 2048, False),    # f16 at exactly 256 vectors: one slot; ranks 5-7 pool nothing
]


def se_case_data(case):
    dt, n, hw, c, ld, r, ldg, _ = case
    rng = np.random.default_rng(R.seed("se", case[1:]))
    x = np.full((n, hw, 1, ld), np.nan, np.float32)
    x[..., :c] = rng.standard_normal((n, hw, 1, c)) + rng.uniform(-1, 1, c)
    x = x.astype(dt)
    w1 = (rng.standard_normal((r, c)) * np.sqrt(2.0 / c)).astype(F32)
    w2 = (rng.standard_normal((c, r)) * np.sqrt(2.0 / r)).astype(F32)
    b1 = rng.uniform(-0.1, 0.1, r).astype(F32)
    b2 = rng.uniform(-0.1, 0.1, c).astype(F32)
    return x, w1, b1, w2, b2


@pytest.mark.parametrize("case", SE_CASES, ids=lambda c: "%s_n%d_hw%d_c%d_ld%d_r%d_ldg%d_%s" % (
    np.dtype(c[0]).name, *c[1:7], "w2off" if c[7] else "w2al"))
def test_se_gate_float_bit_exact(case):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    A, lib = _lib()
    dt, n, hw, c, ld, r, ldg, w2_off = case
    x, w1, b1, w2, b2 = se_case_data(case)
    if n > 16:
        assert n > torch.cuda.get_device_properties(0).multi_processor_count // 8, "images must loop over the clusters"
    d = A.SeGateDesc()
    d.dtype, d.n, d.hw, d.c, d.ld, d.r, d.ldg, d.scale = _dt(dt), n, hw, c, ld, r, ldg, 1.0
    ws = torch.zeros(lib.b200_se_gate_workspace_bytes(d), dtype=torch.uint8, device="cuda")
    assert ws.numel() > 0
    lead = 1 if w2_off else 4                      # W2 starts 4 bytes past a 16-byte boundary, or on one
    wbuf = dev(np.concatenate([np.zeros(lead, F32), w2.ravel()]))
    w2p = C.c_void_p(wbuf.data_ptr() + 4 * lead)
    assert (w2p.value % 16 != 0) == w2_off
    sentinel = np.float32(7.25)
    out = torch.full((n, ldg), float(sentinel), dtype=torch.float32, device="cuda")
    xd, w1d, b1d, b2d = dev(x), dev(w1), dev(b1), dev(b2)
    for _ in range(2):     # a second launch over the same workspace gives the same gate
        A.check(lib.b200_se_gate_run(d, ptr(xd), ptr(w1d), ptr(b1d), w2p, ptr(b2d), ptr(out), ptr(ws), stream_ptr()),
                "se_gate")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    want = S.se_gate_float(x.reshape(n, hw, 1, ld)[..., :c], ld, w1, b1, w2, b2)
    R.assert_same_bits(got[:, :c], want, "gate")
    R.assert_same_bits(got[:, c:], np.full((n, ldg - c), sentinel, F32), "gate padding")
    ref = S.se_gate_f64(x[..., :c].astype(np.float64), w1, b1, w2, b2)
    assert (np.abs(want - ref) <= R.se_gate_bound(x[..., :c], ld, w1, b1, w2, b2)).all()
