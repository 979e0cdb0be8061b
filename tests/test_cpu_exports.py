"""CPU: the argument checks of the interior-tensor export calls that fail before any device is touched, and
api.split_view, which names the parts of a Worker's view result."""
import ctypes as C

import numpy as np
import pytest


def _graph():
    from anakin_b200 import anakin_bin, api, modelzoo
    G = api.Graph.from_bytes(anakin_bin.dumps(modelzoo.build("tiny_resnet", batch=1, precision="int8")))
    G.Optimize()
    return G


def _names(*names):
    return (C.c_char_p * max(1, len(names)))(*[n.encode() if n is not None else None for n in names])


def test_net_create_exports_argument_checks():
    from anakin_b200 import api
    lib = api.load()
    G = _graph()
    out = C.c_void_p()
    cases = [
        ((None, 0, -1, 0, _names("pool5"), 1, C.byref(out)), "null argument"),
        ((G._h, 0, -1, 0, _names("pool5"), 1, None), "null argument"),
        ((G._h, 0, -1, 0, _names("pool5"), -1, C.byref(out)), "negative export count -1"),
        ((G._h, 0, -1, 0, None, 2, C.byref(out)), "null argument"),
        ((G._h, 0, -1, 0, _names("pool5", None), 2, C.byref(out)), "null argument"),
    ]
    for args, msg in cases:
        assert lib.anakin_net_create_exports(*args) != 0
        assert lib.anakin_last_error().decode() == msg, args
        assert not out.value


def test_net_export_calls_on_null_handles():
    from anakin_b200 import api
    lib = api.load()
    nchw = (C.c_int * 4)()
    buf = np.zeros(4, np.float32)
    assert lib.anakin_net_num_exports(None) == 0
    assert lib.anakin_net_export_name(None, 0) is None
    assert lib.anakin_net_export_bytes(None) == 0
    assert lib.anakin_net_export_device_ptr(None, b"pool5") is None
    assert lib.anakin_net_export_info(None, b"pool5", nchw) != 0
    assert lib.anakin_last_error().decode() == "null argument"
    assert lib.anakin_net_read_export(None, b"pool5", buf.ctypes.data_as(C.c_void_p), 4) != 0
    assert lib.anakin_last_error().decode() == "null argument"


def test_worker_create_exports_argument_checks():
    from anakin_b200 import api
    lib = api.load()
    out = C.c_void_p()
    cases = [
        ((None, -2, 1, None, 0, 1, _names("pool5"), 1, C.byref(out)), "null argument"),
        ((b"m.anakin.bin", -2, 1, None, 0, 1, _names("pool5"), -3, C.byref(out)), "negative export count -3"),
        ((b"m.anakin.bin", -2, 1, None, 0, 1, None, 1, C.byref(out)), "null argument"),
        ((b"m.anakin.bin", -2, 1, None, 0, 1, _names(None), 1, C.byref(out)), "null argument"),
    ]
    for args, msg in cases:
        assert lib.anakin_worker_create_exports(*args) != 0
        assert lib.anakin_last_error().decode() == msg, args
        assert not out.value
    assert lib.anakin_worker_output_count(None) == 0


def test_export_kernel_argument_checks():
    from anakin_b200 import saber_abi as A
    lib = A.load()
    x = np.zeros(64, np.float32)
    p = x.ctypes.data_as(C.c_void_p)
    ok = (p, A.UINT8, 1, 2, 2, 4, 16, 0.5, p, None)
    bad = [
        (None,) + ok[1:],
        ok[:8] + (None, None),
        (p, A.INT32) + ok[2:],
        (p, A.UINT8, 0) + ok[3:],
        (p, A.UINT8, 1, 0) + ok[4:],
        (p, A.UINT8, 1, 2, 0) + ok[5:],
        (p, A.UINT8, 1, 2, 2, 0) + ok[6:],
        (p, A.UINT8, 1, 2, 2, 17, 16) + ok[7:],
        (p, A.UINT8, 1, 1 << 16, 1 << 15, 4, 16) + ok[7:],
    ]
    for args in bad:
        assert lib.b200_export_run(*args) == A.INVALID_VALUE, args


def test_split_view_names_the_parts():
    from anakin_b200 import api
    buf = np.arange(4 * 12 + 4 * 8 + 4 * 2 * 3 * 3, dtype=np.float32)
    parts = api.split_view(buf, [("prob", (4, 12)), ("pool5", (4, 8)), ("res", (4, 2, 3, 3))])
    assert list(parts) == ["prob", "pool5", "res"]
    np.testing.assert_array_equal(parts["prob"].reshape(-1), buf[:48])
    np.testing.assert_array_equal(parts["pool5"], buf[48:80].reshape(4, 8))
    np.testing.assert_array_equal(parts["res"], buf[80:].reshape(4, 2, 3, 3))
    assert np.shares_memory(parts["res"], buf)
    parts["pool5"][0, 0] = -1.0
    assert buf[48] == -1.0


@pytest.mark.parametrize("parts,msg", [
    ([("prob", (4, 12)), ("pool5", (4, 7))], "the parts hold 76 floats, the buffer 80"),
    ([("prob", (4, 12)), ("pool5", (4, 9))], "the parts hold 84 floats, the buffer 80"),
    ([("a", (40,)), ("a", (40,))], "a named twice"),
])
def test_split_view_refuses_parts_that_do_not_cover_the_buffer(parts, msg):
    from anakin_b200 import api
    with pytest.raises(api.AnakinError, match=msg):
        api.split_view(np.zeros(80, np.float32), parts)
    with pytest.raises(api.AnakinError, match="float32 buffer"):
        api.split_view(np.zeros(80, np.float64), [("a", (80,))])
