"""GPU: what Net::init makes of every zoo net, pinned against a recording (tests/golden/framework_tables.json.gz).

Net::init chooses a precision per node, an operator per node, each edge's dtype, layout and scale, the conv plans,
the launch schedule and the shared activation memory. A Net is built for every zoo net in fp32, fp16 and (where the zoo
has a calibration table) int8 at batch 2, and this test compares what it reports with the recording:
  * exec_order(), schedule() and launched_ops();
  * tensor_info() of every node of the optimised graph: dims, stored channels, layout, dtype, scale and bytes;
  * activation_bytes() and activation_bytes_unshared();
  * the conv plan lines B200_SABER_VERBOSE=1 prints to stderr;
  * a sha256 of the output of one prediction on seeded inputs.
The memory planner breaks ties between tensors defined at the same step by their addresses, so activation_bytes() may
take one of a few values from one Net to the next (INT8 MobileNet-v1 does): the recording holds every value it saw over
REBUILDS Nets, and a Net must give one of them.

Re-record (on an H100, from the build to be pinned): python tests/test_framework_tables_gpu.py --write
"""
import gzip
import hashlib
import json
import os
import sys

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "framework_tables.json.gz")
NETS = ("tiny_resnet", "tiny_mobilenet", "tiny_se_resnet", "resnet50", "se_resnet50", "mobilenet_v1", "vgg16")
BATCH = 2
REBUILDS = 8


def _precisions(name):
    has_table = os.path.exists(os.path.join(HERE, "golden", "%s_calib.json" % name))
    return ("fp32", "fp16", "int8") if has_table else ("fp32", "fp16")


CASES = [(n, p) for n in NETS for p in _precisions(n)]


def _key(name, precision):
    return "%s-%s" % (name, precision)


def _graph(name, precision):
    from anakin_b200 import anakin_bin, api, modelzoo
    G = api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build(name, batch=1, precision=precision)))
    G.ResetBatchSize("input_0", BATCH)
    G.Optimize()
    return G


def record(name, precision, read_stderr):
    """What Net::init made of the net; read_stderr() returns the stderr written since its last call."""
    import numpy as np
    from anakin_b200 import api, modelzoo
    G = _graph(name, precision)
    read_stderr()
    net = api.Net(G, precision)
    plans = [l for l in read_stderr().splitlines() if l.startswith("[b200_saber] plan")]
    nodes = [d[0] for d in G.describe()]
    c, h, w = G.input_shape("input_0")[1:]
    assert c == 3 and h == w, (c, h, w)
    net.set_input("input_0", modelzoo.synthetic_input(BATCH, h))
    net.prediction()
    net.sync()
    out = net.get_output()
    rec = {
        "exec_order": net.exec_order(),
        "schedule": net.schedule(),
        "launched_ops": net.launched_ops(),
        "tensors": {n: net.tensor_info(n) for n in nodes},
        "activation_bytes": [net.activation_bytes()],
        "activation_bytes_unshared": net.activation_bytes_unshared(),
        "plans": plans,
        "output": [list(out.shape), str(out.dtype), hashlib.sha256(np.ascontiguousarray(out).tobytes()).hexdigest()],
    }
    del net
    for _ in range(REBUILDS - 1):
        rec["activation_bytes"].append(api.Net(G, precision).activation_bytes())
    rec["activation_bytes"] = sorted(set(rec["activation_bytes"]))
    read_stderr()
    return rec


@pytest.fixture(scope="module")
def golden():
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


@pytest.mark.parametrize("name,precision", CASES, ids=[_key(*c) for c in CASES])
def test_net_init_matches_recording(name, precision, golden, capfd, monkeypatch):
    monkeypatch.setenv("B200_SABER_VERBOSE", "1")
    want = golden[_key(name, precision)]
    got = record(name, precision, lambda: capfd.readouterr().err)
    assert set(got["activation_bytes"]) <= set(want["activation_bytes"]), (got["activation_bytes"], want)
    got["activation_bytes"] = want["activation_bytes"]
    for field in want:
        assert got[field] == want[field], field


if __name__ == "__main__" and sys.argv[1:] == ["--write"]:
    import tempfile
    sys.path.insert(0, os.path.dirname(HERE))
    os.environ["B200_SABER_VERBOSE"] = "1"
    # the plan lines come from the device library's stderr: route fd 2 through a file
    log = tempfile.TemporaryFile(mode="w+")
    saved = os.dup(2)
    os.dup2(log.fileno(), 2)

    def read_stderr():
        sys.stderr.flush()
        log.seek(0)
        text = log.read()
        log.seek(0)
        log.truncate()
        return text

    try:
        out = {_key(n, p): record(n, p, read_stderr) for n, p in CASES}
    finally:
        os.dup2(saved, 2)
    with gzip.open(GOLDEN, "wt") as f:
        json.dump(out, f, sort_keys=True)
    print("wrote %d records to %s" % (len(out), GOLDEN))
