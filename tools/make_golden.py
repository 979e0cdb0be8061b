"""Generate the committed fixtures under tests/golden/ with the CPU oracle (run HERE, in the
build container; the GPU box only reads the results):

  <model>_fc_bias.npy  classifier bias b - W.mu (mu = mean penultimate features of the calibration images): centres
                       the logits so that top-1 differs from image to image (modelzoo.center_head)
  <model>_calib.json   max-abs calibration table {node: scale} from the fp32 oracle over 8
                       synthetic images (seeds 1000..1007), CalibrationAlgoType::MAXABS
  <model>_golden.npz   oracle outputs for the bench / parity inputs (seed 42+i): fp32 logits
                       + probabilities, int8 logits + probabilities, top-1 indices

  python tools/make_golden.py [tiny_resnet tiny_mobilenet resnet50 resnet101 vgg16 mobilenet_v1]
  python tools/make_golden.py tiny_se_resnet se_resnet50

The SE nets are walked by tests/se_oracle.py (Axpy and the SE gate). SE-ResNet-50's outputs go to
se_resnet50_ref.npz: bench.py reads <model>_golden.npz with logits node names of its own, which this net does not have.
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from anakin_b200 import modelzoo as Z  # noqa: E402
from oracle import model_walker as MW  # noqa: E402
import se_oracle as SE  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
HW = {"tiny_resnet": 32, "tiny_mobilenet": 32, "tiny_se_resnet": 32}
LOGITS = Z.HEAD_DENSE
INT8_MODELS = {"tiny_resnet", "tiny_mobilenet", "resnet50", "resnet101", "mobilenet_v1", "tiny_se_resnet", "se_resnet50"}
SE_MODELS = {"tiny_se_resnet", "se_resnet50"}
# golden images per model: the batch sizes BASELINE.json's configs name are all covered (C2 b8, C3 b4, C4 b32 -> 4 per
# GPU, C5 b16), ResNet-50 holds 32
IMAGES = {"tiny_resnet": 8, "tiny_mobilenet": 8, "resnet50": 32, "resnet101": 8, "vgg16": 4, "mobilenet_v1": 16,
          "tiny_se_resnet": 8, "se_resnet50": 32}
GOLDEN_NAME = {"se_resnet50": "se_resnet50_ref.npz"}


def _dense_input(vals, g, name):
    node = next(n for n in g["nodes"] if n["name"] == name)
    x = vals[node["ins"][0]]
    if x.ndim == 4:
        x = np.transpose(x, (0, 3, 1, 2))       # Dense flattens in NCHW order
    return np.ascontiguousarray(x).reshape(x.shape[0], -1), node


def main(models):
    os.makedirs(GOLD, exist_ok=True)
    for name in models:
        W = SE if name in SE_MODELS else MW
        fast = {"fast": True} if name == "se_resnet50" else {}   # the AVX-512 arms: bit-identical INT8, re-associated fp32
        hw = HW.get(name, 224)
        nb = IMAGES[name]
        t0 = time.time()
        cal_x = Z.synthetic_input(8, hw, seed=1000)
        # ---- classifier bias that centres the logits (from the UNcentred net)
        g0 = Z.build(name, batch=1, centered=False)
        _, vals = W.run_fp32(g0, cal_x, return_values=True, **fast)
        feat, node = _dense_input(vals, g0, LOGITS[name])
        w = np.asarray(node["attrs"]["weight_1"], np.float32).reshape(int(node["attrs"]["out_dim"]), -1)
        b = np.asarray(node["attrs"]["weight_2"], np.float32).reshape(-1)
        centred = (b.astype(np.float64) - w.astype(np.float64) @ feat.mean(0).astype(np.float64)).astype(np.float32)
        np.save(os.path.join(GOLD, "%s_fc_bias.npy" % name), centred)
        g = Z.build(name, batch=1)                 # picks the new bias up
        x = Z.synthetic_input(nb, hw, seed=42)
        out = {}
        fp32, vals = W.run_fp32(g, x, return_values=True, **fast)
        out["prob_fp32"] = fp32["prob_out"].astype(np.float32)
        out["top1_fp32"] = fp32["prob_out"].argmax(1).astype(np.int32)
        out["logits_fp32"] = vals[LOGITS[name]].reshape(nb, -1).astype(np.float32)
        # what centring took away: logits + logit_offset are the logits of the net with its drawn bias
        out["logit_offset"] = (b - centred).astype(np.float32)
        if name in INT8_MODELS:
            scales = W.calibrate(g, cal_x, **fast)
            with open(os.path.join(GOLD, "%s_calib.json" % name), "w") as f:
                json.dump({"model": name, "algo": "maxabs", "images": 8, "seed": 1000,
                           "edge_scales": {k: float(np.float32(v)) for k, v in scales.items()}}, f, indent=0)
            scales32 = {k: float(np.float32(v)) for k, v in scales.items()}
            q, trace = W.run_int8(g, x, scales32, return_intermediate=True, **fast)
            out["prob_int8"] = q["prob_out"].astype(np.float32)
            out["top1_int8"] = q["prob_out"].argmax(1).astype(np.int32)
            lg = trace[LOGITS[name]][0]
            out["logits_int8"] = lg.reshape(nb, -1).astype(np.float32)
        np.savez_compressed(os.path.join(GOLD, GOLDEN_NAME.get(name, "%s_golden.npz" % name)), **out)
        print("%s: %.1fs, %d images, distinct top-1 fp32 %d%s" % (
            name, time.time() - t0, nb, len(set(out["top1_fp32"].tolist())),
            (" int8 %d (agree with fp32 on %d)" % (len(set(out["top1_int8"].tolist())),
                                                    int((out["top1_int8"] == out["top1_fp32"]).sum()))) if "top1_int8" in out else ""))


if __name__ == "__main__":
    main(sys.argv[1:] or ["tiny_resnet", "tiny_mobilenet", "resnet50", "resnet101", "vgg16", "mobilenet_v1"])
