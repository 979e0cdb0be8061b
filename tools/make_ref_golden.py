"""Record what the reference computes for every case of tests/test_cpu_oracle.py that compares with it, into
tests/golden/ref_oracles.json: arrays as [shape, dtype, SHA-256], scalars and shape lists as values, and the SHA-256 of the
descriptor set built from the reference's .proto files (test_cpu_parser.py). Needs oracle/_ref (`make -C oracle ref`,
built from the reference's sources); the tests then use the records wherever it is absent."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    sys.path.insert(0, ROOT)
    from oracle import pyoracle as O
    O.build(ref=True)
    if O.ref_lib() is None:
        raise SystemExit("oracle/_ref is not built")
    fd, rec = tempfile.mkstemp(suffix=".jsonl")
    os.close(fd)
    env = dict(os.environ, ANAKIN_REF_GOLDEN_RECORD=rec)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(ROOT, "tests", "test_cpu_oracle.py")],
                       cwd=ROOT, env=env)
    out = {}
    with open(rec) as f:
        for line in f:
            d = json.loads(line)
            out[d["key"]] = d["value"]
    os.remove(rec)
    if r.returncode != 0:
        raise SystemExit("the tests failed while recording")
    # the FileDescriptorSet of the reference's .proto files (tests/golden/anakin_proto.desc)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_proto_descriptors import build_descriptor_set
    out["proto_descriptor_set_sha256"] = hashlib.sha256(build_descriptor_set().SerializeToString(deterministic=True)).hexdigest()
    path = os.path.join(ROOT, "tests", "golden", "ref_oracles.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote %s: %d records, %d bytes" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
