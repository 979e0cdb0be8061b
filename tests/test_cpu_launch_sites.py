"""CPU suite: every kernel of the device layer is launched through common.cuh's launch(), which counts the launch
(b200_launch_count, bench.py's gpu_launches) and checks it, and 8-bit codes are written by vec.cuh's one conversion
rule. Both hold only while no source launches or converts on its own, which is what these tests read the sources for."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "anakin_b200", "csrc")


def _code(path):
    with open(path) as f:
        src = f.read()
    return re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", src, flags=re.S))


def _counts(token):
    out = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "**", "*"), recursive=True)):
        if path.endswith((".cu", ".cuh", ".h", ".cpp")):
            n = _code(path).count(token)
            if n:
                out[os.path.relpath(path, CSRC)] = n
    return out


def test_only_the_launch_helper_launches_and_counts():
    assert set(_counts("cudaLaunchKernelEx")) == {"common.cuh"}
    assert set(_counts("count_launch(")) == {"common.cu"}


def test_no_triple_chevron_launch_outside_the_driver_self_test():
    # tensor_map.cu's im2col self-test is a one-time, synchronised probe of the driver and is not counted
    assert _counts("<<<") == {"tensor_map.cu": 1}


def test_8bit_conversion_lives_in_the_codec():
    # the classifier head's pooled codes keep their own u8 / s8 pair (see the comment there)
    assert _counts("cvt.rni.sat") == {"vec.cuh": 2, "fc_stream.cu": 2}


def test_net_launches_the_head_taps_and_join_from_one_site():
    # NetCore's run_eager and profile_ops share one per-entry launch, and calibration statistics and exports share one
    # tap launcher: a second call site would be a second copy of a launch rule, free to drift from the first
    for token in ("b200_head_run(", "b200_calib_stats_run(", "b200_export_run(", "cudaEventRecord(_join_ev"):
        sites = {k: n for k, n in _counts(token).items() if k.startswith("framework" + os.sep)}
        assert sum(sites.values()) == 1, (token, sites)


def test_only_the_conv_planner_reads_the_environment():
    # fusions, streams, the classifier head and the FP32 math kind follow the graph, the shapes and the precision; the
    # planner's knobs stay so that tests and tuning runs can force each conv kernel at chosen shapes
    assert _counts("getenv(") == {"conv_plan.cu": 1}
    assert set(_counts('"B200_SABER_')) == {"conv_plan.cu"}
    assert not _counts('"B200_ANAKIN_')
