"""Device time per replayed prediction of ResNet-50 INT8 with interior-tensor exports (Net(..., exports=[...])).

Cases, at every batch size: no export; pool5 (the 2048-d embedding); pool5 + fc1000 (embedding and logits, both
written behind the fused head); res5c_branch2c (the last ConvEltwise output, [n, 2048, 7, 7], the largest).

For each case a Net is built and its CUDA graph captured; then, for --runs rounds, every case in turn replays --steps
predictions between two CUDA events on its stream. One JSON line per batch and case:
  step_ms       median over the rounds of the mean step time, with min / max
  delta_us      the median minus the no-export case's median
  export_bytes  device bytes of the export buffers; bytes_moved = the exported edge's bytes read + fp32 bytes written
and first a line with the card's name, power limit and maximum SM clock, read in the same run.

  python tools/bench_exports.py [--batches 8,32] [--steps 200] [--runs 7]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from anakin_b200 import anakin_bin, api, modelzoo  # noqa: E402

CASES = {"none": [], "pool5": ["pool5"], "pool5+fc": ["pool5", "fc1000"], "res5c_branch2c": ["res5c_branch2c"]}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers are unlabelled without it, so say so
        return {"name": "unknown", "power_limit": "unknown (%s)" % e}


def bytes_moved(net, nodes):
    total = 0
    for n in nodes:
        info = net.tensor_info(n)
        total += info["bytes"] + 4 * int(np.prod(net.export_info(n)))
    return total


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8,32")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_exports needs a GPU")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for batch in [int(b) for b in a.batches.split(",")]:
        g = modelzoo.build("resnet50", batch=batch, precision="int8")
        G = api.Graph.from_bytes(anakin_bin.dumps(g))
        G.ResetBatchSize("input_0", batch)
        G.Optimize()
        x = modelzoo.synthetic_input(batch)
        nets = {}
        for case, nodes in CASES.items():
            net = api.Net(G, "int8", exports=nodes)
            net.set_input("input_0", x)
            for _ in range(a.warmup):
                net.prediction()
            net.sync()
            assert net.cuda_graph_active(), case
            nets[case] = net
        times = {c: [] for c in CASES}
        for _ in range(a.runs):
            for case, net in nets.items():
                s = torch.cuda.ExternalStream(net.stream)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(s)
                for _ in range(a.steps):
                    net.prediction()
                e1.record(s)
                e1.synchronize()
                times[case].append(e0.elapsed_time(e1) / a.steps)
        base = float(np.median(times["none"]))
        for case, net in nets.items():
            med = float(np.median(times[case]))
            print(json.dumps({"model": "resnet50", "precision": "int8", "batch": batch, "case": case,
                              "exports": CASES[case], "step_ms": round(med, 5),
                              "step_ms_min": round(min(times[case]), 5), "step_ms_max": round(max(times[case]), 5),
                              "delta_us": round(1e3 * (med - base), 2), "export_bytes": net.export_bytes(),
                              "bytes_moved": bytes_moved(net, CASES[case]), "launched_ops": net.launched_ops(),
                              "steps": a.steps, "runs": a.runs}), flush=True)
        del nets


if __name__ == "__main__":
    main()
