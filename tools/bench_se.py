"""ResNet-50 against SE-ResNet-50, INT8, on one GPU: what the squeeze-and-excitation gates cost per step.

  python tools/bench_se.py [--batches 8 32] [--rounds 7] [--reps 20] [--out DIR]

Per batch size: both nets are built (CUDA graph captured), then ROUNDS interleaved rounds each time REPS replays of
each net, every replay behind an L2 flush (a 256 MB memset), device-timed with CUDA events recorded on the net's own
stream around the replay; the median per net is reported. Then profile_ops of the SE net (the 16 SqueezeExcite and 16
AxpyRelu launches), launches_per_step of both nets, and a per-stage breakdown of one gate launch (gate_stages). The card's name, power limit and SM clocks are read in the same run (nvidia-smi query).
One JSON line per batch size; with --out also written to DIR/bench_se.json.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:          # the numbers are still reported, marked as without card data
        return "unavailable (%s)" % e


def _net(model, batch):
    from anakin_b200 import anakin_bin, api, modelzoo
    G = api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build(model, batch=batch, precision="int8")))
    G.ResetBatchSize("input_0", batch)
    G.Optimize()
    net = api.Net(G, "int8")
    net.set_input("input_0", modelzoo.synthetic_input(batch, 224))
    for _ in range(3):
        net.prediction()
    net.sync()
    assert net.cuda_graph_active()
    return net


# (pixels, channels) of branch2c in the four stages of SE-ResNet-50
STAGES = [(56 * 56, 256), (28 * 28, 512), (14 * 14, 1024), (7 * 7, 2048)]


def gate_stages(batch, reps=50):
    """Per-stage breakdown of one SE gate launch (b200_se_gate_run on s8 data of each stage's shape, warm L2): the whole
    launch, and the same launch with one pixel per image, whose time is the cluster's tail (mean, squeeze, excitation)
    alone; the difference is the pooling."""
    import ctypes as C
    import torch
    from anakin_b200 import saber_abi as A
    lib = A.load()
    s = torch.cuda.current_stream()
    out = {}
    for hw, c in STAGES:
        r = c // 16
        res = {}
        for label, pix in (("launch", hw), ("tail", 1)):
            d = A.SeGateDesc()
            d.dtype, d.n, d.hw, d.c, d.ld, d.r, d.ldg, d.scale = A.INT8, batch, pix, c, c, r, c, 0.03
            x = torch.randint(-128, 128, (batch * pix * c,), dtype=torch.int8, device="cuda")
            w = torch.randn(2 * r * c, device="cuda") * 0.05
            b = torch.zeros(r + c, device="cuda")
            g = torch.empty(batch * c, device="cuda")
            ws = torch.zeros(lib.b200_se_gate_workspace_bytes(d), dtype=torch.uint8, device="cuda")
            args = (C.byref(d), C.c_void_p(x.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(b.data_ptr()),
                    C.c_void_p(w.data_ptr() + 4 * r * c), C.c_void_p(b.data_ptr() + 4 * r), C.c_void_p(g.data_ptr()),
                    C.c_void_p(ws.data_ptr()), C.c_void_p(s.cuda_stream))
            for _ in range(5):
                A.check(lib.b200_se_gate_run(*args), "se_gate")
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for _ in range(reps):
                A.check(lib.b200_se_gate_run(*args), "se_gate")
            e1.record(s)
            torch.cuda.synchronize()
            res[label] = 1e3 * e0.elapsed_time(e1) / reps
        res["pooling"] = res["launch"] - res["tail"]
        out["%dx%d" % (hw, c)] = res
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    results = []
    for batch in a.batches:
        nets = {"resnet50": _net("resnet50", batch), "se_resnet50": _net("se_resnet50", batch)}
        times = {k: [] for k in nets}
        streams = {k: torch.cuda.ExternalStream(n.stream) for k, n in nets.items()}
        for _ in range(a.rounds):
            for name, net in nets.items():
                s = streams[name]
                ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.reps)]
                for e0, e1 in ev:
                    flush.zero_()
                    torch.cuda.synchronize()
                    e0.record(s)              # on the net's stream, right around the graph replay
                    net.prediction()
                    e1.record(s)
                    torch.cuda.synchronize()
                times[name].append(float(np.median([e0.elapsed_time(e1) for e0, e1 in ev])))
        se = nets["se_resnet50"]
        prof = se.profile_ops(iters=20)
        gate_us = [t * 1e3 for _, op, t in prof if op == "SqueezeExcite"]
        axpy_us = [t * 1e3 for _, op, t in prof if op in ("Axpy", "AxpyRelu")]
        r = {"batch": batch, "gpu": _gpu_info(),
             "step_ms_median": {k: float(np.median(v)) for k, v in times.items()},
             "step_ms_rounds": times,
             "launches_per_step": {k: int(n.launched_ops()) for k, n in nets.items()},
             "se_gate_us": {"n": len(gate_us), "sum": float(sum(gate_us)), "max": float(max(gate_us))},
             "axpy_us": {"n": len(axpy_us), "sum": float(sum(axpy_us)), "max": float(max(axpy_us))}}
        r["se_cost_us"] = 1e3 * (r["step_ms_median"]["se_resnet50"] - r["step_ms_median"]["resnet50"])
        r["gate_stages_us"] = gate_stages(batch)
        print(json.dumps(r))
        results.append(r)
        del nets, se
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_se.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
