"""GPU parity of the int8 conv plans the planner picks on its own (no forced tile width or split) for the ResNet-50
layer shapes at batch 8: the tile width, split factor and kernel each shape gets, and bit-exact results against the
CPU oracle (x86 Saber semantics)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (n, h, w, c, k, r, stride, pad), residual, expected (kernel, block_n, split)
CASES = [
    ((8, 56, 56, 64, 256, 1, 1, 0), True, ("tile", 64, 1)),       # res2 branch2c: was 256 wide
    ((8, 56, 56, 256, 512, 1, 2, 0), False, (None, 64, 1)),       # res3a branch1: was 128 wide
    ((8, 28, 28, 128, 512, 1, 1, 0), True, (None, 64, 1)),        # res3 branch2c: 392 tiles (per-tile or walker)
    ((8, 14, 14, 1024, 256, 1, 1, 0), False, ("tile", 32, 1)),    # res4 branch2a: 64 wide leaves 52 CTAs
    ((8, 14, 14, 1024, 2048, 1, 2, 0), False, ("tile", 64, 1)),   # res5a branch1: 128 CTAs at 64 wide
    ((8, 14, 14, 256, 256, 3, 1, 1), False, ("slab", 64, 1)),     # res4 branch2b: was a 32-wide slab
    ((8, 7, 7, 512, 512, 3, 1, 1), False, ("tile", 64, 2)),       # res5 branch2b: was a 32-wide slab; 392 = 3 x 128 + 8
    ((8, 7, 7, 512, 512, 3, 1, 1), True, ("tile", 64, 2)),        # the same with a residual
    ((1, 7, 7, 512, 512, 3, 1, 1), False, (None, 32, None)),      # b1: the 32-wide plans stay
]


@pytest.mark.parametrize("case,with_res,expect", CASES)
def test_conv_int8_auto_plan_bit_exact(case, with_res, expect, oracle, monkeypatch):
    for key in ("B200_SABER_FORCE_BN", "B200_SABER_FORCE_SPLIT", "B200_SABER_SLAB", "B200_SABER_PERSISTENT",
                "B200_SABER_SPLIT_MIN_ITERS", "B200_SABER_SPLITK"):
        monkeypatch.delenv(key, raising=False)
    import torch
    from anakin_b200 import saber_abi as A
    from gpu_util import ConvRunner, dev, pad_channels
    n, h, w, c, k, r, stride, pad = case
    rng = np.random.default_rng(hash((case, with_res)) % (2 ** 31))
    x = rng.integers(0, 256, (n, h, w, c)).astype(np.uint8)
    wq = rng.integers(-127, 128, (k, c, r, r)).astype(np.int8)
    bias = rng.uniform(-2000, 2000, k).astype(np.float32)
    scale = rng.uniform(1e-4, 4e-4, k).astype(np.float32)
    kw = dict(stride=(stride, stride), pad=(pad, pad), dil=(1, 1), relu=True)
    oh = oracle.conv_out_size(h, pad, 1, r, stride)
    res = rng.integers(-128, 128, (n, oh, oh, k)).astype(np.int8) if with_res else None
    out_dtype = A.UINT8
    want = oracle.conv_s8_nhwc_x86(x, wq, bias, scale, residual=res, sum_scale=0.5, out_dtype=out_dtype, **kw)
    run = ConvRunner(A.MATH_I8, x.shape, A.UINT8, wq, bias, scale, out_dtype,
                     res_dtype=(A.INT8 if with_res else -1), sum_scale=0.5, ldc=k, **kw)
    info = run.info()
    kernel, bn, split = expect
    got_kernel = "slab" if info["slab"] else ("pers" if info["persistent"] else "tile")
    assert (kernel is None or got_kernel == kernel) and info["block_n"] == bn, info
    assert split is None or info["split"] == split, info
    got = run.run(dev(x), dev(pad_channels(res, k)) if with_res else None)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got.cpu().numpy(), want)
