"""Record the conv plans b200_conv_plan_create builds on the GPU: tests/golden/conv_plans.json.gz (gzip-ed JSON).

  python tools/make_conv_plan_golden.py [--lib anakin_b200/lib/libb200saber.so] [--out tests/golden/conv_plans.json.gz]

A record holds a b200_conv_desc_t, the switches it ran under, the device and its SM count, the status and, on success,
what the plan reports. Only the calls used below are declared (no saber_abi.load()), so any build can be recorded and
two builds compared. Each switch setting is planned in a fresh process: older builds read some switches once.
"""
import argparse
import ctypes as C
import gzip
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from anakin_b200.saber_abi import (FLOAT, HALF, INT8, MATH_F16, MATH_I8, MATH_TF32X3, UINT8,  # noqa: E402
                                   ConvDesc)

SWITCHES = ("B200_SABER_SPLITK", "B200_SABER_FORCE_BN", "B200_SABER_FORCE_SPLIT", "B200_SABER_SLAB",
            "B200_SABER_PERSISTENT", "B200_SABER_VERBOSE")
# switches of older builds; a recording runs with none of them set
RETIRED = ("B200_SABER_SLAB_BN_RULE", "B200_SABER_PERSISTENT_EPI", "B200_SABER_SPLIT_MIN_ITERS",
           "B200_SABER_SMEM_FULL")
FIELDS = [f for f, _ in ConvDesc._fields_]
# math kind -> (input, output, residual) dtypes of the nets
FORMS = {"int8": (MATH_I8, UINT8, UINT8, INT8), "f16": (MATH_F16, HALF, HALF, HALF),
         "tf32x3": (MATH_TF32X3, FLOAT, FLOAT, FLOAT)}


def conv(form, n, h, c, k, r, stride=1, pad=0, res=False, **kw):
    math, in_dt, out_dt, res_dt = FORMS[form]
    d = dict.fromkeys(FIELDS, 0)
    d.update(math=math, in_dtype=in_dt, out_dtype=out_dt, res_dtype=res_dt if res else -1, n=n, h=h, w=h, c=c, k=k,
             ldc=k, r=r, s=r, pad_h=pad, pad_w=pad, stride_h=stride, stride_w=stride, dil_h=1, dil_w=1, relu=1,
             neg_slope=0.0, sum_scale=1.0)
    d.update(kw)
    return d


def fc(form, m, k_in, n_out):
    in_dt = FORMS[form][1]
    out_dt = FLOAT if form != "f16" else HALF
    return conv(form, m, 1, k_in, n_out, 1, relu=0, in_dtype=in_dt, out_dtype=out_dt)


def resnet50_shapes():
    """(name, h_in, c, k, r, stride, pad, residual) of every distinct non-stem conv of ResNet-50."""
    out, h = [], 56
    for si, nblk in enumerate([3, 4, 6, 3]):
        mid, cout, cin = 64 << si, 256 << si, (64 if si == 0 else 128 << si)
        stride = 1 if si == 0 else 2
        ho = h // stride
        tag = "res%d" % (si + 2)
        out += [(tag + "a_branch1", h, cin, cout, 1, stride, 0, False),
                (tag + "a_branch2a", h, cin, mid, 1, stride, 0, False),
                (tag + "_branch2a", ho, cout, mid, 1, 1, 0, False),
                (tag + "_branch2b", ho, mid, mid, 3, 1, 1, False),
                (tag + "_branch2c", ho, mid, cout, 1, 1, 0, True)]
        h = ho
    return out


def cases():
    """(label, desc, switches) of every recorded plan."""
    cs = []
    for form in FORMS:
        for n in (1, 8, 32):
            for name, h, c, k, r, st, pad, res in resnet50_shapes():
                cs.append(("resnet50 %s %s n%d" % (name, form, n), conv(form, n, h, c, k, r, st, pad, res), {}))
    vgg = [(224, 64, 64, True), (112, 64, 128, False), (112, 128, 128, True), (56, 128, 256, False),
           (56, 256, 256, False), (56, 256, 256, True), (28, 256, 512, False), (28, 512, 512, False),
           (28, 512, 512, True), (14, 512, 512, False), (14, 512, 512, True)]
    for form in FORMS:
        for n in (1, 4):
            for h, c, k, pool in vgg:
                extra = dict(fuse_pool=2, pool_stride=2) if pool else {}
                cs.append(("vgg16 %dx%d c%d k%d%s %s n%d" % (h, h, c, k, " pool2" if pool else "", form, n),
                           conv(form, n, h, c, k, 3, 1, 1, **extra), {}))
    mobilenet = [(112, 32, 64), (56, 64, 128), (56, 128, 128), (28, 128, 256), (28, 256, 256), (14, 256, 512),
                 (14, 512, 512), (7, 512, 1024), (7, 1024, 1024)]
    for form in ("int8", "f16"):
        for h, c, k in mobilenet:
            cs.append(("mobilenet_v1 1x1 %dx%d c%d k%d %s n16" % (h, h, c, k, form), conv(form, 16, h, c, k, 1), {}))
    for form in FORMS:
        for k_in, n_out in ((2048, 1000), (4096, 4096)):
            cs.append(("fc %d->%d %s m32" % (k_in, n_out, form), fc(form, 32, k_in, n_out), {}))
    # the int8 plans of tests/test_conv_plan_gpu.py
    for (n, h, w, c, k, r, st, pad), res in [((8, 56, 56, 64, 256, 1, 1, 0), True), ((8, 56, 56, 256, 512, 1, 2, 0), False),
                                              ((8, 28, 28, 128, 512, 1, 1, 0), True), ((8, 14, 14, 1024, 256, 1, 1, 0), False),
                                              ((8, 14, 14, 1024, 2048, 1, 2, 0), False), ((8, 14, 14, 256, 256, 3, 1, 1), False),
                                              ((8, 7, 7, 512, 512, 3, 1, 1), False), ((8, 7, 7, 512, 512, 3, 1, 1), True),
                                              ((1, 7, 7, 512, 512, 3, 1, 1), False)]:
        cs.append(("auto plan n%d %dx%d c%d k%d r%d s%d%s" % (n, h, w, c, k, r, st, " res" if res else ""),
                   conv("int8", n, h, c, k, r, st, pad, res, sum_scale=0.5), {}))
    # every retained switch on a handful of shapes
    probes = [("res4 3x3 int8 n8", conv("int8", 8, 14, 256, 256, 3, 1, 1)),
              ("res4 3x3 tf32x3 n8", conv("tf32x3", 8, 14, 256, 256, 3, 1, 1)),
              ("res5 3x3 int8 n8", conv("int8", 8, 7, 512, 512, 3, 1, 1)),
              ("res5 3x3 f16 n8", conv("f16", 8, 7, 512, 512, 3, 1, 1)),
              ("res2 1x1 res int8 n32", conv("int8", 32, 56, 64, 256, 1, res=True)),
              ("res2 1x1 res f16 n32", conv("f16", 32, 56, 64, 256, 1, res=True)),
              ("res5 1x1 f16 n1", conv("f16", 1, 7, 2048, 512, 1))]
    envs = ([{"B200_SABER_FORCE_BN": str(v)} for v in (32, 64, 128, 256)] +
            [{"B200_SABER_FORCE_SPLIT": str(v)} for v in (1, 2, 4, 8)] +
            [{"B200_SABER_SLAB": v} for v in ("0", "2")] + [{"B200_SABER_PERSISTENT": v} for v in ("0", "2")] +
            [{"B200_SABER_SPLITK": "0"}])
    for env in envs:
        for label, d in probes:
            cs.append(("%s %s" % (label, " ".join("%s=%s" % kv for kv in env.items())), d, env))
    # refusals
    for form in FORMS:
        wrong_in = FLOAT if form in ("int8", "f16") else HALF
        cs += [("refuse %s in_dtype" % form, conv(form, 8, 14, 256, 256, 3, 1, 1, in_dtype=wrong_in), {}),
               ("refuse %s out_dtype" % form, conv(form, 8, 14, 256, 256, 3, 1, 1, out_dtype=INT8 if form != "int8" else HALF), {}),
               ("refuse %s ldc < k" % form, conv(form, 8, 14, 256, 256, 1, ldc=128), {}),
               ("refuse %s pitch" % form, conv(form, 8, 14, 256, 64, 1, ldc=65), {}),
               ("refuse %s channels" % form, conv(form, 8, 14, 3, 64, 3, 1, 1), {}),
               ("refuse %s pad" % form, conv(form, 8, 14, 256, 256, 3, 1, 128), {}),
               ("refuse %s stride" % form, conv(form, 8, 64, 256, 256, 1, 9), {}),
               ("refuse %s dilation" % form, conv(form, 1, 300, 64, 64, 3, 1, 1, dil_h=128, dil_w=128), {}),
               ("refuse %s pool window" % form, conv(form, 4, 48, 64, 64, 3, 1, 1, fuse_pool=12, pool_stride=12), {}),
               ("refuse %s pool residual" % form, conv(form, 4, 28, 64, 64, 3, 1, 1, res=True, fuse_pool=2), {}),
               ("refuse %s pool 1x1" % form, conv(form, 4, 28, 64, 64, 1, fuse_pool=2), {}),
               ("refuse %s pool stride" % form, conv(form, 4, 28, 64, 64, 3, 2, 1, fuse_pool=2), {})]
        if form in ("int8", "f16"):   # an fp32 output over an 8-bit or half residual of a pitch only the output fits
            cs.append(("refuse %s residual pitch" % form,
                       conv(form, 8, 14, 256, 64, 1, res=True, out_dtype=FLOAT, ldc=68), {}))
    cs.append(("refuse unknown math", conv("int8", 8, 14, 256, 256, 1, math=7), {}))
    return cs


def record_group(lib_path, items):
    """Plan every (label, desc, env) of one switch setting in this process; the records as dicts."""
    import torch
    lib, vp, i32 = C.CDLL(lib_path), C.c_void_p, C.c_int32
    for name, res, args in [("b200_conv_packed_weight_bytes", C.c_size_t, [C.POINTER(ConvDesc)]),
                            ("b200_conv_plan_create", C.c_int, [C.POINTER(ConvDesc), vp, vp, vp, C.POINTER(vp)]),
                            ("b200_conv_plan_destroy", None, [vp]),
                            ("b200_conv_plan_info", C.c_int, [vp] + [C.POINTER(i32)] * 5),
                            ("b200_conv_plan_split", C.c_int, [vp]), ("b200_conv_plan_is_slab", C.c_int, [vp]),
                            ("b200_conv_plan_is_persistent", C.c_int, [vp])]:
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    props = torch.cuda.get_device_properties(0)
    out = []
    for label, desc, env in items:
        d = ConvDesc(**desc)
        w = torch.empty(max(int(lib.b200_conv_packed_weight_bytes(C.byref(d))), 16), dtype=torch.uint8, device="cuda")
        plan = vp()
        st = lib.b200_conv_plan_create(C.byref(d), vp(w.data_ptr()), None, None, C.byref(plan))
        rec = {"case": label, "desc": desc, "env": env, "device": props.name, "sms": props.multi_processor_count,
               "status": st}
        if st == -1:
            v = [i32() for _ in range(5)]
            lib.b200_conv_plan_info(plan, *[C.byref(x) for x in v])
            rec.update(zip(("block_n", "grid_x", "grid_y", "k_steps", "smem"), [x.value for x in v]))
            rec.update(split=lib.b200_conv_plan_split(plan), slab=bool(lib.b200_conv_plan_is_slab(plan)),
                       persistent=bool(lib.b200_conv_plan_is_persistent(plan)))
            lib.b200_conv_plan_destroy(plan)
        out.append(rec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "anakin_b200", "lib", "libb200saber.so"))
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "conv_plans.json.gz"))
    ap.add_argument("--group", help=argparse.SUPPRESS)   # internal: plan the cases of one switch setting
    a = ap.parse_args()
    key = lambda case: json.dumps(case[2], sort_keys=True)  # noqa: E731
    if a.group is not None:
        json.dump(record_group(os.path.abspath(a.lib), [c for c in cases() if key(c) == a.group]), sys.stdout)
        return
    by_key = {}
    for k in dict.fromkeys(key(c) for c in cases()):
        env = {n: v for n, v in os.environ.items() if n not in SWITCHES + RETIRED}
        env.update(json.loads(k))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--lib", a.lib, "--group", k], env=env,
                           stdout=subprocess.PIPE, check=True, text=True)
        by_key[k] = iter(json.loads(r.stdout))
    records = [next(by_key[key(c)]) for c in cases()]
    text = "[\n" + ",\n".join(json.dumps(r) for r in records) + "\n]\n"
    with open(a.out, "wb") as f:
        f.write(gzip.compress(text.encode(), compresslevel=9, mtime=0))
    print("%d plans -> %s" % (len(records), a.out))


if __name__ == "__main__":
    main()
