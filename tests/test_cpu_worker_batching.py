"""CPU: the packing decision of a batching Worker (anakin_worker_plan_batch, the same plan_batch the Worker threads call)
on designed queues, and the refusals of anakin_worker_create_batching that come before any device is touched."""
import ctypes as C
import os
import tempfile

import pytest


def plan(sizes, arrive, batch, delay, now):
    """(take, close, deadline_us) of anakin_worker_plan_batch, or (-1, error) when it refuses the queue."""
    from anakin_b200 import api
    lib = api.load()
    n = len(sizes)
    s = (C.c_int * max(1, n))(*sizes)
    a = (C.c_int64 * max(1, n))(*arrive)
    close, deadline = C.c_int(-1), C.c_int64(-1)
    take = lib.anakin_worker_plan_batch(s, a, n, batch, delay, now, C.byref(close), C.byref(deadline))
    if take < 0:
        return take, lib.anakin_last_error().decode()
    return take, bool(close.value), deadline.value


def test_fifo_prefix_that_fits():
    # the batch is a prefix of the queue, in arrival order, while the sizes fit
    assert plan([2, 3, 1], [10, 20, 30], 8, 1000, 40) == (3, False, 1010)
    assert plan([1, 1, 1, 1], [0, 1, 2, 3], 8, 500, 4) == (4, False, 500)


def test_requests_are_never_split():
    # 5 + 4 > 8: the second request is not cut to fill the 3 free slots, it waits, and the batch closes at once
    assert plan([5, 4], [0, 1], 8, 1000, 2) == (1, True, 1000)


def test_oversize_request_waits_for_the_next_batch():
    # the 6 does not fit behind the 3; the 1 queued behind the 6 does not overtake it
    assert plan([3, 6, 1], [0, 1, 2], 8, 1000, 3) == (1, True, 1000)
    # on the next plan the 6 leads, and the 1 joins it
    assert plan([6, 1], [1, 2], 8, 1000, 4) == (2, False, 1001)


def test_full_batch_closes_before_the_window():
    assert plan([4, 4, 2], [0, 1, 2], 8, 1000, 3) == (2, True, 1000)
    assert plan([8], [50], 8, 1000, 50) == (1, True, 1050)
    assert plan([1] * 8, list(range(8)), 8, 10 ** 6, 8) == (8, True, 10 ** 6)


def test_window_closes_a_partial_batch():
    # the deadline runs from the first request's arrival, not the last one's
    assert plan([1, 2], [100, 150], 8, 200, 250) == (2, False, 300)
    assert plan([1, 2], [100, 150], 8, 200, 299) == (2, False, 300)
    assert plan([1, 2], [100, 150], 8, 200, 300) == (2, True, 300)
    assert plan([1, 2], [100, 150], 8, 200, 10 ** 9) == (2, True, 300)


def test_zero_window_takes_only_what_is_queued():
    assert plan([1], [70], 8, 0, 70) == (1, True, 70)
    assert plan([2, 3], [70, 71], 32, 0, 71) == (2, True, 70)


def test_malformed_request_takes_no_slot():
    # size 0 marks a request validation will fail: it is gathered (and fails alone) without using a slot
    assert plan([0, 8], [0, 1], 8, 1000, 2) == (2, True, 1000)
    assert plan([3, 0, 5, 1], [0, 1, 2, 3], 8, 1000, 4) == (3, True, 1000)


def test_empty_queue_and_refusals():
    assert plan([], [], 8, 100, 0) == (0, False, 0)
    assert plan([9], [0], 8, 100, 0) == (-1, "request 0 of 9 images, the batch is 8")
    assert plan([1, -1], [0, 0], 8, 100, 0) == (-1, "request 1 of -1 images, the batch is 8")
    assert plan([1], [0], 0, 100, 0) == (-1, "bad argument")
    assert plan([1], [0], 8, -1, 0) == (-1, "bad argument")


def _names(*names):
    return (C.c_char_p * max(1, len(names)))(*[n.encode() for n in names])


def test_create_batching_refuses_a_negative_window_before_loading():
    from anakin_b200 import api
    lib = api.load()
    out = C.c_void_p()
    # the model path does not exist: the window is refused before anything is read
    for delay in (-1, -1000):
        assert lib.anakin_worker_create_batching(b"missing.anakin.bin", -2, 1, None, 0, 8, None, 0, delay,
                                                 C.byref(out)) != 0
        assert lib.anakin_last_error().decode() == \
            "max_delay_us %d: the batching window must be >= 0" % delay
        assert not out.value
    assert lib.anakin_worker_create_batching(b"missing.anakin.bin", -2, 1, None, 0, 8, _names("pool5"), -2, 0,
                                             C.byref(out)) != 0
    assert lib.anakin_last_error().decode() == "negative export count -2"
    assert lib.anakin_worker_create_batching(None, -2, 1, None, 0, 8, None, 0, 0, C.byref(out)) != 0
    assert lib.anakin_last_error().decode() == "null argument"
    with pytest.raises(api.AnakinError, match="max_delay_us -5: the batching window must be >= 0"):
        api.Worker("missing.anakin.bin", "int8", threads=1, batch=8, max_delay_us=-5)


def test_create_batching_refuses_a_graph_of_two_inputs():
    # the graph is loaded and optimised on the host; the refusal comes before any Net is built
    from anakin_b200 import api, modelzoo
    g = modelzoo.GraphBuilder("TwoInputs")
    a = g.input("input_0", (2, 4, 8, 8))
    b = g.input("input_1", (2, 4, 8, 8))
    g.output("sum_out", g.eltwise_add("sum", a, b))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "two_inputs.anakin.bin")
        modelzoo.save(g.finalize(), path)
        with pytest.raises(api.AnakinError, match="a batching Worker serves graphs of one input; this graph has 2"):
            api.Worker(path, "fp32", threads=1, max_delay_us=0)
