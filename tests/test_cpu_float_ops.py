"""CPU pins of tests/float_ops_ref.py, the references of tests/test_float_ops_gpu.py: the fp32 restatements against the
C oracle, the float64 softmax against scipy, the SE gate's pooling order against float64 within its bound, each
generator's designed edges, and the pooling geometries of tests/test_pointwise_gpu.py (shapes and empty windows)."""
import numpy as np
import pytest

import float_ops_ref as R
import se_oracle as S

F32, F16 = np.float32, np.float16


@pytest.mark.parametrize("op", [R.ELT_PROD, R.ELT_SUM, R.ELT_MAX])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("coef", [(1.0, 1.0), (0.7, -1.3)])
def test_eltwise_restatement_matches_oracle(oracle, op, relu, coef):
    a, b = R.eltwise_edge_block(F32)
    want = oracle.eltwise_f32(a, b, op, coef[0], coef[1], relu)
    R.assert_same_bits(R.eltwise(a, b, op, coef[0], coef[1], relu), want)


@pytest.mark.parametrize("bias", [False, True])
def test_scale_restatement_matches_oracle(oracle, bias):
    """Bit for bit with a bias. Without one the kernel skips the add, so a -0 product stays -0 where the oracle's
    `+ 0.f` gives +0: equal as values, and the only difference."""
    x, w, b = R.scale_data(F32, 40, 24, 24)
    want = oracle.scale_f32(x, 40, 24, 1, w, b if bias else None)
    got = R.scale(x, w, b if bias else None)
    if bias:
        R.assert_same_bits(got, want)
    else:
        np.testing.assert_array_equal(got, want)
        diff = R.same_bits(got, want)
        assert diff.any() and (got[diff] == 0).all() and np.signbit(got[diff]).all()


def test_relu_kinds_match_oracle_where_it_is_exact(oracle):
    """The C oracle's ReLU and ClippedRelu are the kernel's expressions in fp32."""
    x = R.f32_activation_grid()
    for act, slope, coef in ((R.ACT_RELU, 0.0, 0.0), (R.ACT_RELU, 0.1, 0.0), (R.ACT_CLIPPED_RELU, 0.0, 6.0)):
        R.assert_same_bits(R.relu_kinds(x, act, slope, coef), oracle.activation_f32(x, act, slope, coef), str(act))


def test_softmax_f64_matches_scipy():
    from scipy.special import softmax
    for length in R.SOFTMAX_LENGTHS:
        x = R.softmax_bounded_rows(length)
        np.testing.assert_allclose(R.softmax_f64(x), softmax(x.astype(np.float64), axis=-1), rtol=1e-13, atol=1e-300)
    x = np.transpose(R.softmax_bounded_rows(257)[None], (0, 2, 1))
    np.testing.assert_allclose(R.softmax_f64(x, axis=1), softmax(x.astype(np.float64), axis=1), rtol=1e-13, atol=1e-300)


def test_softmax_designed_rows():
    for x, want in R.softmax_exact_rows():
        R.assert_same_bits(R.softmax_f64(x).astype(F32), want)
    for length in R.SOFTMAX_LENGTHS:
        x = R.softmax_bounded_rows(length)
        assert np.isneginf(x[0]).sum() == 1 and (x[0] == x[0].max()).sum() >= 2
        assert np.isfinite(x[1:]).all() and (np.abs(x[1:]) >= 1e30).all()
        assert (np.abs(x[0] - x[0].max()) * R.U > 2.0 ** -22).any(), "x - max must round in e somewhere"
        b = R.softmax_bound(x, R.rows_adds(length))
        assert (b < 1e-5).all()
    # the rows kernel's adds around the 256-thread stride
    assert [R.rows_adds(n) for n in (255, 256, 257, 511)] == [13, 13, 14, 14]


def test_activation_bounds_cover_the_fp32_restatements():
    """The derived bounds hold for an fp32 evaluation of the same formulas in numpy (expf and tanhf replaced by the
    correctly rounded fp32 of the float64 value), and the f16 checker accepts that evaluation."""
    x = R.f32_activation_grid()
    R.assert_activation_f32_edges(x)
    with np.errstate(all="ignore"):
        xf = x.astype(F32)
        e_neg = np.exp(-xf.astype(np.float64)).astype(F32)
        sig = (F32(1) / (e_neg + F32(1))).astype(F32)
        tnh = np.tanh(xf.astype(np.float64)).astype(F32)
        elu = np.where(xf > 0, xf, F32(1.5) * (np.exp(xf.astype(np.float64)).astype(F32) - F32(1))).astype(F32)
    for act, got, coef in ((R.ACT_SIGMOID, sig, 1.0), (R.ACT_TANH, tnh, 1.0), (R.ACT_ELU, elu, 1.5)):
        ratio, bad = R.check_act_f32(got, x, act, coef)
        assert not bad.any() and ratio <= 1, (act, ratio)
    h = R.all_f16_codes()
    with np.errstate(all="ignore"):
        hf = h.astype(F32)
        s16 = (F32(1) / (np.exp(-hf.astype(np.float64)).astype(F32) + F32(1))).astype(F32).astype(F16)
    bad, near, wide, off = R.check_act_f16(s16, h, R.ACT_SIGMOID)
    assert not bad.any() and near.sum() < 655 and not wide.any()
    # ELU's absolute bound near 0 spans several f16 numbers: the codes where the interval is the only check
    wide = R.check_act_f16(h, h, R.ACT_ELU)[2]
    assert wide.any() and (h[wide] <= 0).all() and (h[wide] > -2.0 ** -8).all()


def test_generator_edges():
    R.assert_eltwise_edges(F16)
    R.assert_eltwise_edges(F32)
    for dt in (F16, F32):
        for pixels, c, cs in ((777, 3, 3), (33, 1000, 1008)):
            x, w, b = R.scale_data(dt, pixels, c, cs)
            R.assert_scale_edges(x, w, b, c)
            assert (w[c:] == 0).all() and (b[c:] == 0).all()


def test_se_pooling_order_against_float64():
    """se_mean_ordered is an fp32 sum in the device's order: within gamma(depth) sum|x| / hw + u |m| of the float64
    mean, and different from a plain sequential fp32 sum somewhere (the order is restated, not assumed)."""
    rng = np.random.default_rng(3)
    for dt, n, hw, c, ld in ((F32, 2, 3136, 64, 64), (F16, 3, 49, 96, 104), (F32, 2, 7, 2048, 2048)):
        x = (rng.standard_normal((n, hw, 1, c)) * 10 + 3).astype(dt)
        m = S.se_mean_ordered(x, ld)
        ref = x.astype(np.float64).mean(axis=(1, 2))
        bound = R.gamma(S.se_mean_depth(hw, ld, x.dtype.itemsize)) * np.abs(x.astype(np.float64)).sum(axis=(1, 2)) / hw
        assert (np.abs(m - ref) <= bound + R.U * np.abs(ref)).all()
        if hw > 100:
            seq = np.zeros((n, c), F32)
            for p in range(hw):
                seq = (seq + x[:, p, 0].astype(F32)).astype(F32)
            assert ((seq / F32(hw)).astype(F32) != m).any()
    # slots of the gate CTA: 256 threads over the 16-byte vectors of a pixel
    assert [S.se_slots(ld, es) for ld, es in ((2048, 4), (1024, 4), (72, 4), (104, 2), (2048, 2), (16, 4))] == \
        [1, 1, 14, 19, 1, 64]


def test_se_gate_cases_reach_their_edges():
    from test_float_ops_gpu import SE_CASES, se_case_data
    seen = set()
    for case in SE_CASES:
        dt, n, hw, c, ld, r, ldg, w2_off = case
        chunk = -(-hw // 8)
        seen |= {("slots1" if S.se_slots(ld, np.dtype(dt).itemsize) == 1 else "slots>1"), ("pad" if ld > c else ""),
                 ("empty rank" if (8 - 1) * chunk >= hw else ""), ("loop" if n > 16 else ""),
                 ("scalar r" if r % 4 else ""), ("unaligned" if w2_off and r % 4 == 0 else ""),
                 ("ldg" if ldg > c else ""), dt, hw}
        x, w1, b1, w2, b2 = se_case_data(case)
        assert np.isnan(x[..., c:]).all() and np.isfinite(x[..., :c]).all()
        want = S.se_gate_float(x[..., :c], ld, w1, b1, w2, b2)
        ref = S.se_gate_f64(x[..., :c].astype(np.float64), w1, b1, w2, b2)
        bound = R.se_gate_bound(x[..., :c], ld, w1, b1, w2, b2)
        assert (np.abs(want - ref) <= bound).all() and bound.max() < 1e-3
        assert 0.02 < want.std()
    for need in ("slots1", "slots>1", "pad", "empty rank", "loop", "scalar r", "unaligned", "ldg", F32, F16,
                 1, 7, 49, 3136):
        assert need in seen, need


def _extents(size, window, pad, stride, out):
    """(smallest, largest) window extent along one axis after clipping to [0, size), as pool_window in pointwise.cu."""
    ext = [min(o * stride - pad + window, size) - max(o * stride - pad, 0) for o in range(out)]
    return min(ext), max(ext)


def test_pool_cases_shapes_and_empty_windows(oracle):
    """Every geometry of test_pointwise_gpu.POOL_CASES: the oracle's output size equals b200_pool_out_hw (which runs
    without a GPU), and the smallest window extent along (h, w) is what each case's comment says."""
    import ctypes as C
    from anakin_b200 import saber_abi as A
    from test_pointwise_gpu import POOL_CASES
    lib = A.load()
    min_extent = [(2, 2), (2, 2), (2, 2), (2, 2), (7, 7), (1, 1), (17, 17), (0, 0), (-1, -1), (-1, -1), (0, 0), (2, 2),
                  (3, 3), (1, 3), (3, 2), (1, 1)]
    assert len(min_extent) == len(POOL_CASES)
    for case, want_ext in zip(POOL_CASES, min_extent):
        n, h, w, c, win, pad, stride, glob, floor = case
        d = A.PoolDesc()
        d.dtype, d.type, d.n, d.h, d.w, d.c = A.FLOAT, 1, n, h, w, c
        d.window_h, d.window_w = win
        d.pad_h, d.pad_w = pad
        d.stride_h, d.stride_w = stride
        d.global_pooling, d.floor_as_conv = int(glob), int(floor)
        oh, ow = C.c_int32(), C.c_int32()
        assert lib.b200_pool_out_hw(C.byref(d), C.byref(oh), C.byref(ow)) == A.SUCCESS
        if glob:
            win, pad, stride = (h, w), (0, 0), (h, w)
        want = oracle.pool_out_size(h, w, win[0], win[1], pad[0], pad[1], stride[0], stride[1], glob, floor)
        assert (oh.value, ow.value) == want, case
        got_ext = (_extents(h, win[0], pad[0], stride[0], oh.value)[0], _extents(w, win[1], pad[1], stride[1], ow.value)[0])
        assert got_ext == want_ext, (case, got_ext)
        if floor:
            assert oracle.pool_out_size(h, w, win[0], win[1], pad[0], pad[1], stride[0], stride[1], glob, False) != want
    taps = {c[4][0] * c[4][1] for c in POOL_CASES if not c[7]}
    assert {15, 16} <= taps


@pytest.mark.parametrize("ptype", [1, 2, 3])
@pytest.mark.parametrize("unsigned", [False, True])
def test_pool_oracle_empty_windows(oracle, ptype, unsigned):
    """Over an empty window the 8-bit oracle writes code 0 (MAX and AVG: a sum of no taps), whatever the input."""
    x = np.full((2, 21, 24, 16), 255 if unsigned else -128, np.uint8 if unsigned else np.int8)
    got = oracle.pool_s8_nhwc(x, (2, 2), (0, 0), (3, 3), ptype)
    assert got.shape == (2, 8, 9, 16)
    assert (got[:, 7] == 0).all() and (got[:, :, 8] == 0).all()
    assert (got[:, :7, :8] == x[0, 0, 0, 0]).all()
