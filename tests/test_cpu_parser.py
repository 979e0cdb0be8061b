"""CPU suite: the hand-written .anakin.bin codecs against a CANONICAL protobuf implementation.

google.protobuf message classes are built from a FileDescriptorSet derived from the reference's own four .proto
files (tools/make_proto_descriptors.py -> tests/golden/anakin_proto.desc; re-derived and compared when
/root/reference is present). With them:
  * what the Python writer (anakin_b200/anakin_bin.py) and the C++ writer (Graph::save, csrc/framework/graph.cpp)
    emit is byte-for-byte what protobuf's serialiser emits for the same message, up to the order of map entries
    (protobuf leaves map order unspecified; every record -- node, attribute value, tensor, edge list -- is compared
    as bytes);
  * what protobuf serialises -- including encodings the hand-written writers never produce (unpacked repeated
    fields, explicit oneof zeros, unknown fields) -- is read identically by the C++ parser;
  * shared weight tensors (TensorProto.shared / share_from, model_io.cpp:147-151) and INT8 weight payloads
    (CacheDate.c, model_io.cpp:204-216) load, run through Optimize and round-trip through Graph::save;
  * a tensor whose payload does not fill its shape is rejected instead of being zero-filled.
"""
import hashlib
import json
import os
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
DESC = os.path.join(ROOT, "tests", "golden", "anakin_proto.desc")


@pytest.fixture(scope="module")
def pb():
    from make_proto_descriptors import message_classes
    with open(DESC, "rb") as f:
        return message_classes(f.read())


def _records(buf, nested=(2,)):
    """Multiset of a message's (field, wire type, payload bytes) records; records of the `nested` fields (NodeProto
    inside GraphProto) are themselves reduced to multisets, so that only map-entry ORDER is forgotten."""
    from anakin_b200.anakin_bin import _fields
    out = []
    for field, wt, v in _fields(memoryview(buf)):
        payload = bytes(v) if wt == 2 else v
        if wt == 2 and field in nested:
            payload = _records(payload, nested=())
        out.append((field, wt, payload))
    return tuple(sorted(out, key=repr))


def _same_up_to_map_order(a, b):
    return len(a) == len(b) and _records(a) == _records(b)


def _cpp_save(blob, optimize=False):
    from anakin_b200 import api
    G = api.Graph.from_bytes(blob)
    if optimize:
        G.Optimize()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "m.anakin.bin")
        G.save(p)
        with open(p, "rb") as f:
            return f.read()


def test_descriptor_fixture_matches_the_reference_protos():
    """The fixture is the FileDescriptorSet built from the reference's four .proto files: its SHA-256 as built from
    them is stored in tests/golden/ref_oracles.json (tools/make_ref_golden.py); where those sources are present the
    set is rebuilt and compared byte for byte."""
    with open(DESC, "rb") as f:
        data = f.read()
    with open(os.path.join(os.path.dirname(DESC), "ref_oracles.json")) as f:
        want = json.load(f)["proto_descriptor_set_sha256"]
    assert hashlib.sha256(data).hexdigest() == want
    from make_proto_descriptors import PROTO_DIR, build_descriptor_set
    if os.path.isdir(PROTO_DIR):
        assert build_descriptor_set().SerializeToString(deterministic=True) == data


@pytest.mark.parametrize("model,precision", [("tiny_resnet", "int8"), ("tiny_resnet", "fp32"), ("tiny_mobilenet", "int8")])
def test_writers_are_byte_identical_to_protobuf(pb, model, precision):
    from anakin_b200 import anakin_bin, modelzoo
    g = modelzoo.build(model, batch=2, precision=precision)
    blob = anakin_bin.dumps(g)
    msg = pb["GraphProto"]()
    msg.ParseFromString(blob)
    assert len(msg.nodes) == len(g["nodes"])
    canon = msg.SerializeToString(deterministic=True)
    assert _same_up_to_map_order(blob, canon), "Python writer differs from protobuf's encoding"
    cpp = _cpp_save(blob)
    assert _same_up_to_map_order(cpp, canon), "C++ Graph::save differs from protobuf's encoding"
    # and the optimised graph (merged attrs, fused nodes) is valid, canonical protobuf too
    opt = _cpp_save(blob, optimize=True)
    m2 = pb["GraphProto"]()
    m2.ParseFromString(opt)
    assert m2.summary.is_optimized and len(m2.nodes) < len(msg.nodes)
    assert _same_up_to_map_order(opt, m2.SerializeToString(deterministic=True))


def test_cpp_parser_reads_what_protobuf_writes(pb):
    """Build the message with protobuf alone, using encodings our writers never emit."""
    G = pb["GraphProto"]()
    G.name = "pbnet"
    n = G.nodes.add()
    n.name = "input_0"
    n.Op.name = "Input"
    n.outs.append("fc")
    n.attr["input_shape"].cache_list.i.extend([1, 8, 1, 1])
    n.attr["input_shape"].cache_list.type = 4
    n.attr["input_shape"].cache_list.size = 4
    n.attr["input_shape"].type = 30
    n = G.nodes.add()
    n.name = "fc"
    n.Op.name = "Dense"
    n.ins.append("input_0")
    n.outs.append("out")
    n.attr["axis"].i = 1
    n.attr["axis"].type = 4
    n.attr["out_dim"].i = 0          # oneof member explicitly set to zero: protobuf emits it
    n.attr["out_dim"].type = 4
    n.attr["bias_term"].b = False
    n.attr["bias_term"].type = 20
    w = np.arange(32, dtype=np.float32).reshape(4, 8) / 7
    t = n.attr["weight_1"].tensor
    t.shape.dim.value.extend([1, 1, 4, 8])
    t.shape.dim.size = 4
    t.valid_shape.dim.value.extend([1, 1, 4, 8])
    t.valid_shape.dim.size = 4
    t.data.f.extend(w.ravel().tolist())
    t.data.type = 13
    t.data.size = 32
    n.attr["weight_1"].type = 31
    n = G.nodes.add()
    n.name = "out"
    n.Op.name = "Output"
    n.ins.append("fc")
    G.edges_in["fc"].target.add(node="input_0", scale=[0.5], layout=8)
    G.edges_out["input_0"].target.add(node="fc", scale=[0.5], layout=8)
    G.edges_in["out"].val.append("fc")
    G.edges_out["fc"].val.append("out")
    G.ins.append("input_0")
    G.outs.append("out")
    G.version.major = 2
    blob = G.SerializeToString()
    from anakin_b200 import anakin_bin
    back = pb["GraphProto"]()
    back.ParseFromString(_cpp_save(blob))
    assert back.nodes[1].attr["out_dim"].type == 4 and back.nodes[1].attr["out_dim"].i == 0
    np.testing.assert_array_equal(np.array(back.nodes[1].attr["weight_1"].tensor.data.f, np.float32), w.ravel())
    assert list(back.edges_in["fc"].target[0].scale) == [0.5]
    assert list(back.nodes[0].attr["input_shape"].cache_list.i) == [1, 8, 1, 1]
    # the Python reader agrees
    g = anakin_bin.loads(blob)
    np.testing.assert_array_equal(np.asarray(g["nodes"][1]["attrs"]["weight_1"]).ravel(), w.ravel())


def _two_dense_graph(second_weight):
    from anakin_b200 import anakin_bin
    w = (np.arange(32, dtype=np.float32).reshape(1, 1, 4, 8) - 11) / 5

    def dense(name, src, dst, weight):
        return {"name": name, "op": "Dense", "ins": [src], "outs": [dst],
                "attrs": {"axis": 1, "out_dim": 4, "bias_term": False, "weight_1": weight}}
    nodes = [
        {"name": "input_0", "op": "Input", "ins": [], "outs": ["fc_a", "fc_b"], "attrs": {"input_shape": [1, 8, 1, 1]}},
        dense("fc_a", "input_0", "out_a", w),
        dense("fc_b", "input_0", "out_b", second_weight),
        {"name": "out_a", "op": "Output", "ins": ["fc_a"], "outs": [], "attrs": {}},
        {"name": "out_b", "op": "Output", "ins": ["fc_b"], "outs": [], "attrs": {}},
    ]
    g = {"name": "shared", "nodes": nodes, "ins": ["input_0"], "outs": ["out_a", "out_b"],
         "edges_in": {"fc_a": [("input_0", None)], "fc_b": [("input_0", None)], "out_a": [("fc_a", None)],
                      "out_b": [("fc_b", None)]},
         "edges_out": {"input_0": [("fc_a", None), ("fc_b", None)], "fc_a": [("out_a", None)], "fc_b": [("out_b", None)]}}
    return anakin_bin.dumps(g), w


def test_shared_weight_tensors_resolve_and_round_trip(pb):
    blob, w = _two_dense_graph({"share_from": "fc_a"})
    saved = _cpp_save(blob)
    m = pb["GraphProto"]()
    m.ParseFromString(saved)
    by = {n.name: n for n in m.nodes}
    assert by["fc_b"].attr["weight_1"].tensor.shared and by["fc_b"].attr["weight_1"].tensor.share_from == b"fc_a"
    assert len(by["fc_b"].attr["weight_1"].tensor.data.f) == 0        # a reference, not a copy
    np.testing.assert_array_equal(np.array(by["fc_a"].attr["weight_1"].tensor.data.f, np.float32), w.ravel())
    assert _same_up_to_map_order(saved, m.SerializeToString(deterministic=True))
    from anakin_b200 import api
    with pytest.raises(api.AnakinError, match="does not own"):
        api.Graph.from_bytes(_two_dense_graph({"share_from": "nowhere"})[0])


def test_int8_weight_payload_round_trips(pb):
    q = (np.arange(32, dtype=np.int32).reshape(1, 1, 4, 8) * 7 % 255 - 127).astype(np.int8)
    blob, _ = _two_dense_graph({"tensor": q, "scale": [0.5, 0.25, 0.125, 1.0]})
    m = pb["GraphProto"]()
    m.ParseFromString(_cpp_save(blob))
    t = {n.name: n for n in m.nodes}["fc_b"].attr["weight_1"].tensor
    assert t.data.type == 2 and t.data.size == 32 and len(t.data.f) == 0
    np.testing.assert_array_equal(np.frombuffer(t.data.c, np.int8), q.ravel())
    assert list(t.scale.f) == [0.5, 0.25, 0.125, 1.0]
    from anakin_b200 import anakin_bin
    back = anakin_bin.loads(_cpp_save(blob))
    v = {n["name"]: n for n in back["nodes"]}["fc_b"]["attrs"]["weight_1"]
    assert v["tensor"].dtype == np.int8 and v["scale"] == [0.5, 0.25, 0.125, 1.0]


def test_payload_size_mismatch_is_rejected(pb):
    from anakin_b200 import api
    blob, _ = _two_dense_graph(np.zeros((1, 1, 4, 8), np.float32))
    m = pb["GraphProto"]()
    m.ParseFromString(blob)
    t = {n.name: n for n in m.nodes}["fc_b"].attr["weight_1"].tensor
    del t.data.f[20:]
    with pytest.raises(api.AnakinError, match="payload holds 20 elements"):
        api.Graph.from_bytes(m.SerializeToString())
