"""GPU: the FP16 and FP32 kernels bit for bit on designed data whose sums are exact (tests/float_exact.py).

With exact sums the only roundings are + bias, * neg_slope and the store, so every conv path, split-K factor, tile
width, residual type and f16 store must give the oracle's bits exactly, and the f16 stores numpy's round-half-to-even
conversion of them. Covered:
- dense exact data through the im2col kernel at every tile width, split-K 2 / 4 / 8, the slab kernel, the persistent
  kernel and the slab kernel's fused MAX pooling, with f16 and fp32 outputs and residuals; padding channels past k keep
  a sentinel;
- the float epilogue grid: f16 ties of both signs and directions, +-1 fp32 ulp around them, overflow at 65520, f16
  subnormal ties, -0.0 out of the relu and the (acc + res) + bias order;
- the 3xTF32 terms (Ahi Whi + Alo Whi + Ahi Wlo, without Alo Wlo), and the tensor core's truncation of the low plane;
- the stem (f16 staging rounds half to even), fc_stream's f16 and fp32 stores, the fp32 depthwise kernels, the f16
  layout transform and f16 average pooling on ties;
- identical bits on two runs of every float split-K plan and of the persistent kernel.
"""
import ctypes as C

import numpy as np
import pytest

import float_exact as F
from anakin_b200 import saber_abi as A
from test_conv_gpu import PERSISTENT_CASES, POOL_CASES, SLAB_CASES, SPLIT_CASES

pytestmark = pytest.mark.gpu

SENTINEL = -777.0
_UINT = {2: np.uint16, 4: np.uint32}


def _torch_dt(dt):
    import torch
    return torch.float16 if dt == A.HALF else torch.float32


def assert_bits(got, want, info=None):
    """Equal bit patterns (so -0.0 differs from 0.0, and inf must match inf)."""
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.shape == want.shape, (got.shape, want.shape)
    assert got.dtype == want.dtype, (got.dtype, want.dtype)
    gb, wb = got.view(_UINT[got.itemsize]), want.view(_UINT[want.itemsize])
    bad = np.argwhere(gb != wb)
    assert bad.shape[0] == 0, "%d of %d differ, first %s: got %s want %s (info %s)" % (
        bad.shape[0], got.size, bad[:5].tolist(), got[tuple(bad[:5].T)], want[tuple(bad[:5].T)], info)


def max_bn(out_dt, res_dt):
    return 128 if out_dt == A.FLOAT or res_dt == A.FLOAT else 256


def use_kernel(monkeypatch, kernel, bn=0, split=0):
    """tileN: the im2col kernel at width N; slab; persistent (unsplit plans only)."""
    if kernel == "im2col":
        monkeypatch.setenv("B200_SABER_SLAB", "0")
        monkeypatch.setenv("B200_SABER_PERSISTENT", "0")
    elif kernel == "slab":
        monkeypatch.setenv("B200_SABER_SLAB", "2")
    else:
        monkeypatch.setenv("B200_SABER_PERSISTENT", "2")
        monkeypatch.setenv("B200_SABER_SLAB", "0")
        monkeypatch.setenv("B200_SABER_FORCE_SPLIT", "1")
    if bn:
        monkeypatch.setenv("B200_SABER_FORCE_BN", str(bn))
    if split:
        monkeypatch.setenv("B200_SABER_FORCE_SPLIT", str(split))


def run_conv(math, x, w, bias, out_dt, res=None, res_dt=None, relu=True, neg_slope=0.1, stride=(1, 1), pad=(0, 0),
             dil=(1, 1), out=None, **kw):
    """One plan on designed data into a sentinel-filled output whose row pitch exceeds k: (output [..., :k], info)."""
    import torch
    from gpu_util import ConvRunner, dev, pad_channels
    k = w.shape[0]
    ldc = F.ldc_for(k, out_dt, res_dt if res is not None else None)
    run = ConvRunner(F.MATH[math], x.shape, F.IN_DT[math], w, bias, None, out_dt,
                     res_dtype=res_dt if res is not None else -1, sum_scale=1.0, ldc=ldc, stride=stride, pad=pad,
                     dil=dil, relu=relu, neg_slope=neg_slope, **kw)
    info = run.info()
    if out is None:
        out = torch.full((x.shape[0], run.ho, run.wo, ldc), SENTINEL, dtype=_torch_dt(out_dt), device="cuda")
    run.run(dev(x), dev(pad_channels(res, ldc)) if res is not None else None, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert (got[..., k:] == SENTINEL).all(), "padding channels past k must keep the sentinel (info %s)" % info
    return got[..., :k], info


def dense_run(case, variant, **kw):
    math, out_dt, res_dt = F.DENSE_VARIANTS[variant]
    n, h, w, c, k, r, s, stride, ph, pw, dil = F.full_geom(case)
    x, wt, bias, res, want = F.dense_case(case, variant)
    from gpu_util import pad_channels
    xin = pad_channels(x, F.in_channels(math, c, r)[1])
    got, info = run_conv(math, xin, wt, bias, out_dt, res, res_dt, stride=(stride, stride), pad=(ph, pw),
                         dil=(dil, dil), **kw)
    return got, want, info


VARIANTS = list(F.DENSE_VARIANTS)
WIDTHS = [32, 64, 128, 256]


# ================================================================================ 1. dense exact data, every conv path
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("case", F.DENSE_F_CASES)
def test_dense_im2col(case, variant, monkeypatch):
    """The im2col kernel; the tile width rotates over the (case, variant) grid so every width meets every kind."""
    _, out_dt, res_dt = F.DENSE_VARIANTS[variant]
    bn = WIDTHS[(F.DENSE_F_CASES.index(case) + VARIANTS.index(variant)) % 4]
    bn = min(bn, max_bn(out_dt, res_dt))
    use_kernel(monkeypatch, "im2col", bn=bn)
    got, want, info = dense_run(case, variant)
    assert info["block_n"] == bn and not info["slab"] and not info["persistent"], info
    assert_bits(got, want, info)


@pytest.mark.parametrize("variant", ["f16_h", "f16_h_res-h"])
def test_dense_im2col_256_ragged(variant, monkeypatch):
    """The 256-wide tile, which only 2-byte outputs and residuals take, with k = 200 ragged against it."""
    use_kernel(monkeypatch, "im2col", bn=256)
    got, want, info = dense_run(F.DENSE_F_CASES[-1], variant)
    assert info["block_n"] == 256, info
    assert_bits(got, want, info)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("case,bn,split", SPLIT_CASES)
def test_dense_split_k(case, bn, split, variant, monkeypatch):
    use_kernel(monkeypatch, "im2col", bn=bn, split=split)
    got, want, info = dense_run(case, variant)
    assert (info["block_n"], info["split"]) == (bn, split) and not info["slab"], info
    assert_bits(got, want, info)


SLAB_BNS = [0, 32, 64, 128, 256]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("case", SLAB_CASES)
def test_dense_slab(case, variant, monkeypatch):
    """5x5, 1x7, 7x1, images wider than one tile; the forced width rotates (0: the planner's). Filters wider or taller
    than 3 taps are forced to at most 64 channels: the slab planner leaves some wider tiles of them to the im2col
    kernel."""
    _, out_dt, res_dt = F.DENSE_VARIANTS[variant]
    n, h, w, c, k, r, s, ph, pw = case
    bn = min(SLAB_BNS[(SLAB_CASES.index(case) + VARIANTS.index(variant)) % 5], max_bn(out_dt, res_dt),
             64 if max(r, s) > 3 else 256)
    use_kernel(monkeypatch, "slab", bn=bn)
    got, want, info = dense_run((n, h, w, c, k, r, s, 1, ph, pw, 1), variant)
    assert info["slab"] and (not bn or info["block_n"] == bn), info
    assert_bits(got, want, info)


@pytest.mark.parametrize("variant", [v for v in VARIANTS if not v.startswith("tf32x3")])
@pytest.mark.parametrize("case", PERSISTENT_CASES)
def test_dense_persistent(case, variant, monkeypatch):
    n, h, w, c, k, r, stride, pad = case
    # the planner's 256-wide tiles (2-byte outputs and residuals) stay on the per-tile kernel
    use_kernel(monkeypatch, "persistent", bn=128 if k >= 128 else 0)
    got, want, info = dense_run((n, h, w, c, k, r, stride, pad, 1), variant)
    assert info["persistent"] and not info["slab"], info
    assert_bits(got, want, info)


def test_persistent_refuses_tf32x3(monkeypatch):
    """The persistent kernel has no tf32x3 instance: a tf32x3 plan stays on the per-tile im2col kernel, and is exact."""
    use_kernel(monkeypatch, "persistent")
    case = PERSISTENT_CASES[0]
    n, h, w, c, k, r, stride, pad = case
    got, want, info = dense_run((n, h, w, c, k, r, stride, pad, 1), "tf32x3_f_res-f")
    assert not info["persistent"] and not info["slab"], info
    assert_bits(got, want, info)


FUSED_POOL_CASES = [POOL_CASES[0], POOL_CASES[3], POOL_CASES[4], (1, 20, 22, 64, 200, 3, 1, 3, 2, 0)]


@pytest.mark.parametrize("variant", ["f16_h", "f16_f", "tf32x3_f"])
@pytest.mark.parametrize("case", FUSED_POOL_CASES)
def test_dense_fused_max_pool(case, variant, oracle, monkeypatch):
    """The slab kernel's fused MAX pooling. With k = 200 and 128-wide tiles the last n-tile's tf32x3 high-image load
    reads rows of the low image into channels >= k: the 16-byte pooled stores must drop them."""
    n, h, w, c, k, r, pad, pk, ps, pp = case
    if k == 200:
        monkeypatch.setenv("B200_SABER_FORCE_BN", "128")
    _, out_dt, _ = F.DENSE_VARIANTS[variant]
    x, wt, bias, _, conv = F.dense_case((n, h, w, c, k, r, 1, pad, 1), variant)
    want = oracle.pool_f32(conv.astype(np.float32), (pk, pk), (pp, pp), (ps, ps), A.POOL_MAX, nhwc=True)
    want = want.astype(conv.dtype)
    got, info = run_conv(variant.split("_")[0], x, wt, bias, out_dt, pad=(pad, pad), fuse_pool=pk, pool_stride=ps,
                         pool_pad=pp)
    assert info["slab"] and (k != 200 or info["block_n"] == 128), info
    assert_bits(got, want, info)


def test_float_plans_refuse_types_their_epilogue_cannot_store():
    """Half outputs and residuals belong to the f16 kind, 8-bit ones to the int8 kind: anything else is refused with
    INVALID_VALUE rather than left unwritten. The accepted combinations, built with the same shape and arguments, show
    that the refusals come from the type checks."""
    from gpu_util import ConvRunner
    w = np.ones((32, 32, 1, 1), np.float32)

    def plan(math, in_dt, out_dt, res_dt):
        wt = w.astype(np.float16) if in_dt == A.HALF else (w.astype(np.int8) if in_dt == A.INT8 else w)
        return ConvRunner(math, (1, 8, 8, 32), in_dt, wt, None, np.ones(32, np.float32) if math == A.MATH_I8 else None,
                          out_dt, res_dtype=res_dt, ldc=64)

    good = [(A.MATH_TF32X3, A.FLOAT, A.FLOAT, A.FLOAT), (A.MATH_TF32X3, A.FLOAT, A.FLOAT, -1),
            (A.MATH_F16, A.HALF, A.HALF, A.HALF), (A.MATH_F16, A.HALF, A.FLOAT, A.FLOAT),
            (A.MATH_I8, A.INT8, A.INT8, A.UINT8), (A.MATH_I8, A.INT8, A.FLOAT, -1)]
    for combo in good:
        plan(*combo)
    bad = [(A.MATH_TF32X3, A.FLOAT, A.HALF, -1), (A.MATH_TF32X3, A.FLOAT, A.FLOAT, A.HALF), (A.MATH_F16, A.HALF, A.INT8, -1),
           (A.MATH_F16, A.HALF, A.HALF, A.UINT8),
           (A.MATH_I8, A.INT8, A.HALF, -1), (A.MATH_I8, A.INT8, A.INT8, A.FLOAT)]
    for combo in bad:
        with pytest.raises(A.SaberError, match="conv_plan_create failed: SaberInvalidValue"):
            plan(*combo)


# ================================================================================ 2. float epilogue grid
GRID_KERNELS = ["tile32", "tile64", "tile128", "tile256", "slab", "persistent"]


@pytest.mark.parametrize("kernel", GRID_KERNELS)
@pytest.mark.parametrize("variant", list(F.GRID_VARIANTS))
def test_float_epilogue_grid(variant, kernel, monkeypatch):
    math, out_dt, res_dt, relu, slope = F.GRID_VARIANTS[variant]
    x, bias, res, want = F.grid_case(variant)
    r = 1
    if kernel.startswith("tile"):
        bn = int(kernel[4:])
        if bn > max_bn(out_dt, res_dt):
            pytest.skip("4-byte outputs and residuals cap the tile at 128 channels")
        use_kernel(monkeypatch, "im2col", bn=bn)
    elif kernel == "persistent" and math == "tf32x3":
        pytest.skip("the persistent kernel refuses tf32x3 (test_persistent_refuses_tf32x3)")
    else:
        use_kernel(monkeypatch, kernel)
        r = 3 if kernel == "slab" else 1
    w = F.grid_weights(r)
    if math == "f16":
        x, w = x.astype(np.float16), w.astype(np.float16)
    got, info = run_conv(math, x, w, bias, out_dt, res, res_dt, relu=relu, neg_slope=slope, pad=(r // 2, r // 2))
    if kernel.startswith("tile"):
        assert info["block_n"] == bn and not info["slab"] and not info["persistent"], info
    else:
        assert info[kernel], info
    assert_bits(got, want, info)


# ================================================================================ 3./4. 3xTF32 terms, low-plane truncation
# (case, kernel, bn, split); case = (n, h, w, c, k, r, s, stride, pad)
X3_RUNS = [
    ((1, 14, 14, 128, 200, 3, 3, 1, 1), "im2col", 32, 1),
    ((1, 14, 14, 128, 200, 3, 3, 1, 1), "im2col", 64, 2),
    ((1, 14, 14, 128, 200, 3, 3, 1, 1), "im2col", 128, 4),
    ((1, 14, 14, 128, 200, 3, 3, 1, 1), "im2col", 128, 8),
    ((2, 9, 9, 256, 72, 1, 1, 1, 0), "im2col", 64, 1),
    ((1, 12, 30, 64, 200, 3, 3, 1, 1), "slab", 128, 0),
    ((1, 12, 30, 64, 200, 3, 3, 1, 1), "slab", 64, 0),
]


@pytest.mark.parametrize("math", ["tf32x3"])
@pytest.mark.parametrize("case,kernel,bn,split", X3_RUNS)
def test_split_terms(case, kernel, bn, split, math, monkeypatch):
    """Exactly Ahi Whi + Alo Whi + Ahi Wlo with the kernels' split."""
    n, h, w, c, k, r, s, stride, pad = case
    use_kernel(monkeypatch, kernel, bn=bn, split=split)
    x, wt, bias, want = F.x3_case(case)
    got, info = run_conv(math, x, wt, bias, A.FLOAT, relu=False, stride=(stride, stride), pad=(pad, pad))
    if kernel == "im2col":
        assert (info["block_n"], info["split"]) == (bn, split) and not info["slab"], info
    else:
        assert info[kernel] and (not bn or info["block_n"] == bn), info
    assert_bits(got, want, info)


def test_split_terms_truncate_low_plane():
    """wgmma .tf32 truncates the 13-bit low parts of the activations to 11 significant bits, as the split relies on:
    Ahi Whi + trunc(Alo) Whi + Ahi Wlo."""
    x, wt, bias, want = F.x3_trunc_case()
    got, info = run_conv("tf32x3", x, wt, bias, A.FLOAT, relu=False)
    assert_bits(got, want, info)


@pytest.mark.parametrize("math", ["tf32x3"])
def test_split_terms_fused_pool(math, oracle, monkeypatch):
    monkeypatch.setenv("B200_SABER_FORCE_BN", "128")
    case = (1, 12, 30, 64, 200, 3, 3, 1, 1)
    x, wt, bias, conv = F.x3_case(case)
    want = oracle.pool_f32(conv, (3, 3), (0, 0), (2, 2), A.POOL_MAX, nhwc=True)
    got, info = run_conv(math, x, wt, bias, A.FLOAT, relu=False, pad=(1, 1), fuse_pool=3, pool_stride=2)
    assert info["slab"] and info["block_n"] == 128, info
    assert_bits(got, want, info)


# ================================================================================ 5. stem
STEM_CASES = [(2, 3, 40, 44, 64, 7, 7, 2, 3, (3, 2, 0)), (1, 3, 33, 33, 16, 5, 5, 2, 2, (3, 2, 1)),
              (1, 3, 30, 34, 48, 3, 3, 1, 1, None)]


@pytest.mark.parametrize("monotone", [0, 1])
@pytest.mark.parametrize("math", ["f16", "tf32x3"])
@pytest.mark.parametrize("case", STEM_CASES, ids=["7x7s2-pool", "5x5s2-padpool", "3x3s1"])
def test_stem_exact(case, math, monotone, oracle):
    """f16: fp32 inputs on f16 half-ulp ties, converted at staging with round half to even; f16 outputs bit for bit.
    tf32x3: the staging split."""
    from test_stem_gpu import _run_stem, _stem_desc
    n, c, h, w, k, r, s, stride, pad, pool = case
    if monotone and pool is None:
        pytest.skip("the flag only matters with a fused pooling")
    x, w_op, bias, want = F.stem_case(case, math)
    out_dt = A.HALF if math == "f16" else A.FLOAT
    if pool is not None:
        pk = ((pool[0],) * 2, (pool[2],) * 2, (pool[1],) * 2)
        want = oracle.pool_f32(want.astype(np.float32), *pk, A.POOL_MAX, nhwc=True).astype(want.dtype)
    d = _stem_desc(A, F.MATH[math], out_dt, case, F.ldc_for(k, out_dt), True, 1.0, neg_slope=0.1, monotone=monotone)
    got = _run_stem(A, d, x, w_op, bias, None, _torch_dt(out_dt), fill=SENTINEL)
    assert (got[..., k:] == SENTINEL).all(), "padding channels past k must keep the sentinel"
    assert_bits(got[..., :k], want)


# ================================================================================ 6. fc_stream
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("out", [A.HALF, A.FLOAT], ids=["f16out", "f32out"])
@pytest.mark.parametrize("math", ["f32", "f16"])
@pytest.mark.parametrize("k", [1024, 25088])
def test_fc_stream_exact(k, math, out, relu):
    """Every row count the kernel takes, one to 16; columns past n_out keep the sentinel."""
    import torch
    from gpu_util import dev, ptr, stream_ptr
    x, w, bias, want = F.fc_case(k, math, out, relu)
    lib = A.load()
    n = w.shape[0]
    xd, wd, bd = dev(x), dev(w), dev(bias)
    for m in range(1, 17):
        d = A.FcStreamDesc()
        d.math, d.in_dtype = (A.MATH_F16, A.HALF) if math == "f16" else (A.MATH_TF32X3, A.FLOAT)
        d.out_dtype = out
        d.m, d.k, d.ldx, d.n_out, d.ldo = m, k, k, n, n + 8
        d.relu, d.neg_slope = int(relu), 0.1
        o = torch.full((m, d.ldo), SENTINEL, dtype=_torch_dt(out), device="cuda")
        A.check(lib.b200_fc_stream_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), None, ptr(o), stream_ptr()), "fc_stream")
        torch.cuda.synchronize()
        got = o.cpu().numpy()
        assert (got[:, n:] == SENTINEL).all(), "columns past n_out must keep the sentinel (m %d)" % m
        assert_bits(got[:, :n], want[:m], "m %d" % m)


# ================================================================================ 7. depthwise f32
# fp32 3x3 stride 1 takes the tiled kernel from 28 x 28 outputs on, the row kernel below that
DW_EXACT = {"row-3x3": (2, 14, 14, 32, 3, 1, 1), "row-3x3s2": (2, 28, 28, 32, 3, 2, 1), "vec-5x5": (2, 28, 28, 32, 5, 1, 1),
            "vec-3x3d2": (2, 28, 28, 32, 3, 1, 2), "tile-8": (2, 30, 37, 32, 3, 1, 1), "tile-4": (1, 29, 70, 16, 3, 1, 1)}


@pytest.mark.parametrize("kernel", list(DW_EXACT))
def test_dwconv_f32_exact(kernel):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    n, h, w, c, r, stride, dil = DW_EXACT[kernel]
    x, wt, bias, want = F.dw_case(n, h, w, c, r, stride, dil)
    pad = (r - 1) * dil // 2
    d = A.ConvDesc()
    d.math, d.in_dtype, d.out_dtype, d.res_dtype = A.MATH_TF32X3, A.FLOAT, A.FLOAT, -1
    d.n, d.h, d.w, d.c, d.k, d.ldc, d.r, d.s = n, h, w, c, c, c, r, r
    d.pad_h = d.pad_w = pad
    d.stride_h = d.stride_w = stride
    d.dil_h = d.dil_w = dil
    d.relu, d.neg_slope = 1, 0.1
    wrsc = np.ascontiguousarray(np.transpose(wt[:, 0], (1, 2, 0)))
    xd, wd, bd = dev(x), dev(wrsc), dev(bias)
    out = torch.full(want.shape, SENTINEL, dtype=torch.float32, device="cuda")
    A.check(A.load().b200_dwconv_run(C.byref(d), ptr(xd), ptr(wd), ptr(bd), None, ptr(out), stream_ptr()))
    torch.cuda.synchronize()
    assert_bits(out.cpu().numpy(), want)


# ================================================================================ 8. layout transform and pooling ties
@pytest.mark.parametrize("shape", [(2, 3, 17, 9), (2, 40, 5, 7)], ids=["c3-pixel-kernel", "c40-transpose-kernel"])
def test_nchw_to_nhwc_f16_ties(shape):
    import torch
    from gpu_util import dev, ptr, stream_ptr
    n, c, h, w = shape
    x = F.f16_tie_inputs(shape, np.random.default_rng(31))
    F.assert_tie_inputs(x, at_least=5)
    want = np.ascontiguousarray(x.transpose(0, 2, 3, 1)).astype(np.float16)
    c_pad = (c + 15) // 16 * 16
    out = torch.full((n, h, w, c_pad), 5.0, dtype=torch.float16, device="cuda")
    xd = dev(x)
    A.check(A.load().b200_nchw_to_nhwc(ptr(xd), ptr(out), A.HALF, n, c, h, w, c_pad, 1.0, stream_ptr()))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert_bits(got[..., :c], want)
    assert (got[..., c:] == 0).all()


@pytest.mark.parametrize("ptype", [A.POOL_AVG_INC, A.POOL_AVG_EXC], ids=["avg_inc", "avg_exc"])
@pytest.mark.parametrize("geom", [(2, 0, 2, False), (8, 0, 8, True), (4, 0, 2, False)], ids=["2x2s2", "global8x8", "4x4s2"])
def test_pool_f16_average_ties(geom, ptype, oracle):
    """Checkerboards of adjacent f16 values: every even window's fp32 mean is an exact f16 tie."""
    from test_pointwise_gpu import _pool
    win, pad, stride, glob = geom
    n, h, w, c = 2, 8, 8, 64
    x = F.pool_tie_planes(n, h, w, c)
    mean = oracle.pool_f32(x.astype(np.float32), (win, win), (pad, pad), (stride, stride), ptype, nhwc=True,
                           global_pooling=glob)
    tie, up = F.f16_ties(mean)
    assert tie.mean() > 0.9 and up.any() and (~up).any()
    got = _pool(A.HALF, (n, h, w, c, win, pad, stride, glob), ptype, x)
    assert_bits(got, mean.astype(np.float16))


# ================================================================================ 9. determinism
@pytest.mark.parametrize("math", ["f16", "tf32x3"])
@pytest.mark.parametrize("case,bn,split", SPLIT_CASES)
def test_split_k_deterministic(case, bn, split, math, monkeypatch):
    """The split-K reduction has a fixed summation order: random data, the same bits on two runs into the same buffers."""
    use_kernel(monkeypatch, "im2col", bn=bn, split=split)
    _deterministic(case, math, (bn, split))


@pytest.mark.parametrize("math", ["f16"])
@pytest.mark.parametrize("case", PERSISTENT_CASES[:3])
def test_persistent_deterministic(case, math, monkeypatch):
    use_kernel(monkeypatch, "persistent")
    n, h, w, c, k, r, stride, pad = case
    _deterministic((n, h, w, c, k, r, stride, pad, 1), math, None)


def _deterministic(case, math, expect):
    import torch
    n, h, w, c, k, r, stride, pad, dil = case
    rng = np.random.default_rng(F.seed(case, math))
    dt = np.float16 if math == "f16" else np.float32
    x = rng.uniform(-1, 1, (n, h, w, c)).astype(dt)
    wt = rng.standard_normal((k, c, r, r)).astype(dt)
    bias = rng.uniform(-1, 1, k).astype(np.float32)
    res = rng.uniform(-1, 1, (n, (h + 2 * pad - r) // stride + 1, (w + 2 * pad - r) // stride + 1, k)).astype(np.float32)
    kw = dict(stride=(stride, stride), pad=(pad, pad))
    first, info = run_conv(math, x, wt, bias, A.FLOAT, res, A.FLOAT, **kw)
    if expect is not None:
        assert (info["block_n"], info["split"]) == expect, info
    else:
        assert info["persistent"], info
    out = torch.full((n,) + first.shape[1:3] + (F.ldc_for(k, A.FLOAT, A.FLOAT),), SENTINEL, dtype=torch.float32,
                     device="cuda")
    a, _ = run_conv(math, x, wt, bias, A.FLOAT, res, A.FLOAT, out=out, **kw)
    b, _ = run_conv(math, x, wt, bias, A.FLOAT, res, A.FLOAT, out=out, **kw)
    assert_bits(a, first, info)
    assert_bits(b, first, info)
