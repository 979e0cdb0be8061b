"""Python front end over the framework C ABI (include/anakin_b200.h, libanakin_b200.so).

Mirrors the reference's user API names (Graph.load / ResetBatchSize / Optimize / save,
Net.init / prediction / get_in / get_out -- examples/cuda/example_nv_cnn_net.cpp:21-71) for
tests and bench.py.  All compute happens in the native libraries; there is no Python or
CPU fallback path.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# ANAKIN_B200_LIBDIR: alternative directory holding both .so files (A/B experiments between builds)
_LIBDIR = os.environ.get("ANAKIN_B200_LIBDIR") or os.path.join(_HERE, "lib")
LIB_PATH = os.path.join(_LIBDIR, "libanakin_b200.so")

FP32, FP16, INT8 = 0, -1, -2
PRECISIONS = {"fp32": FP32, "fp16": FP16, "int8": INT8}
_NP_OF_DTYPE = {0: np.float16, 1: np.float32, 3: np.int8, 7: np.uint8}

_vp, _i, _sz, _cp = C.c_void_p, C.c_int, C.c_size_t, C.c_char_p


class ImageFormat(C.Structure):
    """anakin_image_format_t: network channel i = (image channel src_channel[i] - mean[i]) * scale[i] (fp32, no FMA)."""
    _fields_ = [("src_channel", C.c_int32 * 4), ("mean", C.c_float * 4), ("scale", C.c_float * 4)]


SYMBOLS = {
    "anakin_graph_set_input_image": (_i, [_vp, _cp, C.POINTER(ImageFormat)]),
    "anakin_graph_input_image": (_i, [_vp, _cp, C.POINTER(ImageFormat)]),
    "anakin_graph_input_shape": (_i, [_vp, _cp, C.POINTER(_i)]),
    "anakin_net_set_input_image": (_i, [_vp, _cp, _vp, _sz]),
    "anakin_worker_sync_prediction_image": (_i, [_vp, _vp, _sz, _vp, _sz]),
    "anakin_worker_async_prediction_image": (_i, [_vp, _vp, _sz, _vp, _sz]),
    "anakin_graph_set_input_image_resize": (_i, [_vp, _cp, _i, _i, _i]),
    "anakin_graph_input_image_resize": (_i, [_vp, _cp, C.POINTER(_i), C.POINTER(_i), C.POINTER(_i)]),
    "anakin_net_set_input_images": (_i, [_vp, _cp, _vp, _sz, _vp, _sz]),
    "anakin_worker_sync_prediction_images": (_i, [_vp, _vp, _sz, _vp, _sz, _vp, _sz]),
    "anakin_worker_async_prediction_images": (_i, [_vp, _vp, _sz, _vp, _sz, _vp, _sz]),
    "anakin_last_error": (_cp, []),
    "anakin_graph_load": (_i, [_cp, C.POINTER(_vp)]),
    "anakin_graph_load_buffer": (_i, [_vp, _sz, C.POINTER(_vp)]),
    "anakin_graph_reset_batch_size": (_i, [_vp, _cp, _i]),
    "anakin_graph_reshape": (_i, [_vp, _cp, C.POINTER(_i)]),
    "anakin_graph_optimize": (_i, [_vp, _i]),
    "anakin_graph_save": (_i, [_vp, _cp]),
    "anakin_graph_describe": (_sz, [_vp, _vp, _sz]),
    "anakin_graph_destroy": (None, [_vp]),
    "anakin_net_create": (_i, [_vp, _i, _i, C.POINTER(_vp)]),
    "anakin_net_num_inputs": (_i, [_vp]),
    "anakin_net_num_outputs": (_i, [_vp]),
    "anakin_net_input_name": (_cp, [_vp, _i]),
    "anakin_net_output_name": (_cp, [_vp, _i]),
    "anakin_net_tensor_info": (_i, [_vp, _cp, C.POINTER(_i), C.POINTER(_i), C.POINTER(_i), C.POINTER(_i),
                                    C.POINTER(C.c_float), C.POINTER(_sz)]),
    "anakin_net_tensor_device_ptr": (_vp, [_vp, _cp]),
    "anakin_net_set_input": (_i, [_vp, _cp, _vp, _sz]),
    "anakin_net_prediction": (_i, [_vp]),
    "anakin_net_sync": (_i, [_vp]),
    "anakin_net_read_tensor": (_i, [_vp, _cp, _vp, _sz]),
    "anakin_net_stream": (_vp, [_vp]),
    "anakin_net_launched_ops": (_i, [_vp]),
    "anakin_net_cuda_graph_active": (_i, [_vp]),
    "anakin_net_set_cuda_graph": (_i, [_vp, _i]),
    "anakin_net_exec_order": (_sz, [_vp, _vp, _sz]),
    "anakin_net_activation_bytes": (_sz, [_vp]),
    "anakin_net_activation_bytes_unshared": (_sz, [_vp]),
    "anakin_net_weight_ptrs": (_i, [_vp, C.POINTER(_vp), _i]),
    "anakin_weight_arena_stats": (_sz, [C.POINTER(_sz), C.POINTER(_sz), C.POINTER(_sz)]),
    "anakin_weight_arena_set_receive": (None, [C.c_int]),
    "anakin_weight_arena_flat_bytes": (_sz, [C.c_int]),
    "anakin_weight_arena_export": (C.c_int, [C.c_int, _vp, _sz]),
    "anakin_weight_arena_import": (C.c_int, [C.c_int, _vp, _sz]),
    "anakin_net_create_ex": (_i, [_vp, _i, _i, _i, C.POINTER(_vp)]),
    "anakin_net_profile_ops": (_i, [_vp, _i, _i, C.POINTER(C.c_float), _i]),
    "anakin_net_destroy": (None, [_vp]),
    "anakin_worker_create": (_i, [_cp, _i, _i, C.POINTER(_i), _i, _i, C.POINTER(_vp)]),
    "anakin_worker_sync_prediction": (_i, [_vp, _vp, _sz, _vp, _sz]),
    "anakin_worker_wait_ready": (_i, [_vp]),
    "anakin_worker_async_prediction": (_i, [_vp, _vp, _sz, _vp, _sz]),
    "anakin_worker_async_get_result": (_i, [_vp]),
    "anakin_worker_destroy": (None, [_vp]),
}

_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libanakin_b200.so is not built (%s); run `python -m anakin_b200.build`. "
                           "There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class AnakinError(RuntimeError):
    pass


def _check(rc, what):
    if rc != 0:
        raise AnakinError("%s: %s" % (what, load().anakin_last_error().decode()))


def _text(fn, handle):
    n = fn(handle, None, 0)
    buf = C.create_string_buffer(n + 1)
    fn(handle, buf, n + 1)
    return buf.value.decode()


def pack_images(images):
    """(pixels, hw) of a request on an image input with on-device resize: the uint8 [h_i, w_i, c] arrays packed back
    to back (rows unpadded) and the int32 [count, 2] array of their (h_i, w_i)."""
    arrs = [np.ascontiguousarray(a) for a in images]
    for a in arrs:
        if a.dtype != np.uint8 or a.ndim != 3:
            raise AnakinError("images: uint8 [h, w, c] arrays expected, got %s %s" % (a.dtype, a.shape))
    pix = np.concatenate([a.reshape(-1) for a in arrs]) if arrs else np.zeros(0, np.uint8)
    hw = np.array([a.shape[:2] for a in arrs], np.int32).reshape(-1, 2)
    return pix, hw


class Graph:
    """graph::Graph<NV, P> (load / ResetBatchSize / Reshape / Optimize / save)."""

    def __init__(self):
        self._h = _vp()
        self._lib = load()

    @staticmethod
    def from_file(path):
        g = Graph()
        _check(g._lib.anakin_graph_load(path.encode(), C.byref(g._h)), "Graph.load(%s)" % path)
        return g

    @staticmethod
    def from_bytes(data):
        g = Graph()
        buf = C.create_string_buffer(data, len(data))
        _check(g._lib.anakin_graph_load_buffer(buf, len(data), C.byref(g._h)), "Graph.load(buffer)")
        return g

    def ResetBatchSize(self, in_name, batch):
        _check(self._lib.anakin_graph_reset_batch_size(self._h, in_name.encode(), batch), "ResetBatchSize")

    def Reshape(self, in_name, shape):
        arr = (_i * 4)(*shape)
        _check(self._lib.anakin_graph_reshape(self._h, in_name.encode(), arr), "Reshape")

    def input_shape(self, in_name):
        """[N, C, H, W] of Input node in_name."""
        arr = (_i * 4)()
        _check(self._lib.anakin_graph_input_shape(self._h, in_name.encode(), arr), "input_shape")
        return list(arr)

    def Optimize(self, with_fusion=True):
        _check(self._lib.anakin_graph_optimize(self._h, int(with_fusion)), "Optimize")

    def save(self, path):
        _check(self._lib.anakin_graph_save(self._h, path.encode()), "save")

    def set_input_image(self, name, mean, scale, src_channel=None):
        """Declare Input `name` an 8-bit image input: uint8 [n, h, w, c] interleaved pixels, c = the Input's channel
        count, and network channel i = (image channel src_channel[i] - mean[i]) * scale[i] in fp32 (numpy's
        (u.astype(np.float32) - mean) * scale). src_channel defaults to the identity; [2, 1, 0] swaps BGR and RGB.
        The lists must have exactly one entry per channel of the Input."""
        mean, scale = list(mean), list(scale)
        src = list(range(len(mean))) if src_channel is None else list(src_channel)
        lens = (len(mean), len(scale), len(src))
        shape = (_i * 4)()      # (an unknown name / a non-Input node is reported by the C call below)
        c = shape[1] if self._lib.anakin_graph_input_shape(self._h, name.encode(), shape) == 0 else None
        if len(set(lens)) != 1 or lens[0] > 4 or (c is not None and lens[0] != c):
            raise AnakinError("set_input_image(%s): mean, scale and src_channel need one entry per channel of the Input "
                              "(%s, at most 4), got %d, %d, %d" % ((name, c) + lens))
        f = ImageFormat()
        for i in range(4):
            # (entries past the lists are invalid: the C side checks the first c)
            f.src_channel[i] = int(src[i]) if i < len(src) else -1
            f.mean[i] = float(mean[i]) if i < len(mean) else float("nan")
            f.scale[i] = float(scale[i]) if i < len(scale) else float("nan")
        _check(self._lib.anakin_graph_set_input_image(self._h, name.encode(), C.byref(f)), "set_input_image")

    def input_image(self, name):
        """{"src_channel", "mean", "scale"} (one entry per channel) of an image input, or None for an fp32 input."""
        f = ImageFormat()
        if not self._lib.anakin_graph_input_image(self._h, name.encode(), C.byref(f)):
            return None
        c = sum(1 for s in f.src_channel if s >= 0)     # entries past the channel count read -1
        return {"src_channel": list(f.src_channel)[:c], "mean": list(f.mean)[:c], "scale": list(f.scale)[:c]}

    def set_input_image_resize(self, name, max_h, max_w, resize_short=0):
        """Let the image input `name` (set_input_image first) take images of any size up to max_h x max_w, resized and
        centre-cropped on the GPU to the Input's H x W: short side to resize_short (at least max(H, W)) then centre
        crop, or a stretch to H x W when resize_short is 0. Requests then go through Net.set_input_images /
        Worker.*_prediction_images."""
        _check(self._lib.anakin_graph_set_input_image_resize(self._h, name.encode(), int(max_h), int(max_w),
                                                             int(resize_short)), "set_input_image_resize")

    def input_image_resize(self, name):
        """{"max_h", "max_w", "resize_short"} of an image input with on-device resize, or None."""
        v = [_i(), _i(), _i()]
        if not self._lib.anakin_graph_input_image_resize(self._h, name.encode(), *[C.byref(x) for x in v]):
            return None
        return {"max_h": v[0].value, "max_w": v[1].value, "resize_short": v[2].value}

    def describe(self):
        """[(name, op, [ins], [outs])] in execution order."""
        out = []
        for line in _text(self._lib.anakin_graph_describe, self._h).splitlines():
            name, op, ins, outs = line.split("|")
            out.append((name, op, [s for s in ins.split(",") if s], [s for s in outs.split(",") if s]))
        return out

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.anakin_graph_destroy(self._h)
            self._h = _vp()


class Net:
    """Net<NV, P>: init(graph) on a device, prediction(), tensors by node name."""

    def __init__(self, graph, precision="fp32", device=-1, keep_edges=False):
        """keep_edges=True gives every edge tensor its own buffer so intermediate tensors can be read back after
        prediction() (parity tests); the default shares buffers between edges whose live ranges do not overlap."""
        self._lib = load()
        self._h = _vp()
        prec = PRECISIONS[precision] if isinstance(precision, str) else precision
        _check(self._lib.anakin_net_create_ex(graph._h, prec, device, 1 if keep_edges else 0, C.byref(self._h)),
               "Net.init")
        self.in_names = [self._lib.anakin_net_input_name(self._h, i).decode()
                         for i in range(self._lib.anakin_net_num_inputs(self._h))]
        self.out_names = [self._lib.anakin_net_output_name(self._h, i).decode()
                          for i in range(self._lib.anakin_net_num_outputs(self._h))]

    def tensor_info(self, node):
        dims = (_i * 4)()
        cs, layout, dtype = _i(), _i(), _i()
        scale, nbytes = C.c_float(), _sz()
        _check(self._lib.anakin_net_tensor_info(self._h, node.encode(), dims, C.byref(cs), C.byref(layout),
                                                C.byref(dtype), C.byref(scale), C.byref(nbytes)), "tensor_info")
        return {"dims": list(dims), "c_stored": cs.value, "layout": layout.value, "dtype": dtype.value,
                "scale": scale.value, "bytes": nbytes.value}

    def device_ptr(self, node):
        return self._lib.anakin_net_tensor_device_ptr(self._h, node.encode())

    def set_input(self, name, host_nchw):
        a = np.ascontiguousarray(host_nchw, np.float32)
        self._keep = a
        _check(self._lib.anakin_net_set_input(self._h, name.encode(), a.ctypes.data_as(_vp), a.size), "set_input")

    def set_input_ptr(self, name, host_ptr, count):
        _check(self._lib.anakin_net_set_input(self._h, name.encode(), _vp(host_ptr), count), "set_input")

    def set_input_image(self, name, images_nhwc):
        """8-bit images [n, h, w, c] (uint8, interleaved) into an image input (Graph.set_input_image)."""
        a = np.ascontiguousarray(images_nhwc)
        if a.dtype != np.uint8:
            raise AnakinError("set_input_image(%s): uint8 pixels expected, got %s" % (name, a.dtype))
        self._keep = a
        _check(self._lib.anakin_net_set_input_image(self._h, name.encode(), a.ctypes.data_as(_vp), a.nbytes),
               "set_input_image")

    def set_input_images(self, name, images):
        """A request on an image input with on-device resize: a list of uint8 [h_i, w_i, c] arrays, one per image of
        the batch, each of its own size. They are packed back to back and copied to the GPU asynchronously."""
        pix, hw = pack_images(images)
        self._keep = (pix, hw)
        _check(self._lib.anakin_net_set_input_images(self._h, name.encode(), pix.ctypes.data_as(_vp), pix.nbytes,
                                                     hw.ctypes.data_as(_vp), hw.shape[0]), "set_input_images")

    def prediction(self):
        _check(self._lib.anakin_net_prediction(self._h), "prediction")

    def sync(self):
        _check(self._lib.anakin_net_sync(self._h), "sync")

    def read_tensor(self, node):
        """Raw storage of a node's output as numpy: NHWC tensors come back [n,h,w,c_stored]."""
        info = self.tensor_info(node)
        n, c, h, w = info["dims"]
        dt = _NP_OF_DTYPE[info["dtype"]]
        shape = (n, h, w, info["c_stored"]) if info["layout"] == 9 else (n, c, h, w)
        out = np.empty(shape, dt)
        assert out.nbytes == info["bytes"], (out.nbytes, info)
        _check(self._lib.anakin_net_read_tensor(self._h, node.encode(), out.ctypes.data_as(_vp), out.nbytes),
               "read_tensor")
        return out, info

    def read_tensor_into(self, node, host_ptr, nbytes):
        _check(self._lib.anakin_net_read_tensor(self._h, node.encode(), _vp(host_ptr), nbytes), "read_tensor")

    def get_output(self, name=None):
        """fp32 output as [N, C] (or NCHW) numpy."""
        name = name or self.out_names[0]
        arr, info = self.read_tensor(name)
        n, c, h, w = info["dims"]
        if info["layout"] == 9:
            arr = arr[..., :c]
            arr = arr.reshape(n, c) if h == 1 and w == 1 else np.transpose(arr, (0, 3, 1, 2))
        else:
            arr = arr.reshape(n, c) if h == 1 and w == 1 else arr
        return np.ascontiguousarray(arr)

    @property
    def stream(self):
        return self._lib.anakin_net_stream(self._h)

    def launched_ops(self):
        return self._lib.anakin_net_launched_ops(self._h)

    def cuda_graph_active(self):
        return bool(self._lib.anakin_net_cuda_graph_active(self._h))

    def set_cuda_graph(self, enable):
        _check(self._lib.anakin_net_set_cuda_graph(self._h, int(enable)), "set_cuda_graph")

    def exec_order(self):
        return [l.split(":") for l in _text(self._lib.anakin_net_exec_order, self._h).splitlines()]

    def profile_ops(self, iters=5, reps=1):
        """[(node, op, ms)] device time per launched op (eager, CUDA-event pair per op; reps > 1 =
        that many back-to-back launches per pair, i.e. steady-state time)."""
        order = self.exec_order()
        buf = (C.c_float * len(order))()
        _check(self._lib.anakin_net_profile_ops(self._h, iters, reps, buf, len(order)), "profile_ops")
        return [(n, o, float(buf[i])) for i, (n, o) in enumerate(order)]

    def activation_bytes(self):
        return self._lib.anakin_net_activation_bytes(self._h)

    def activation_bytes_unshared(self):
        return self._lib.anakin_net_activation_bytes_unshared(self._h)

    def weight_ptrs(self):
        n = self._lib.anakin_net_weight_ptrs(self._h, None, 0)
        buf = (_vp * max(1, n))()
        self._lib.anakin_net_weight_ptrs(self._h, buf, n)
        return [int(buf[i] or 0) for i in range(n)]

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.anakin_net_destroy(self._h)
            self._h = _vp()


def weight_arena_stats():
    """(device bytes, entries, hits, misses) of the process-wide packed-weight arena."""
    lib = load()
    e, h, m = _sz(), _sz(), _sz()
    b = lib.anakin_weight_arena_stats(C.byref(e), C.byref(h), C.byref(m))
    return int(b), e.value, h.value, m.value


def weight_arena_set_receive(on):
    """Receive mode: Nets initialised while it is on allocate their packed-weight images without building them; the
    images then arrive with weight_arena_import (multi-GPU replicas, see anakin_b200/dist.py)."""
    load().anakin_weight_arena_set_receive(1 if on else 0)


def weight_arena_flat_bytes(device):
    return int(load().anakin_weight_arena_flat_bytes(device))


def weight_arena_export(device, dev_ptr, nbytes):
    _check(load().anakin_weight_arena_export(device, _vp(dev_ptr), nbytes), "weight_arena_export")


def weight_arena_import(device, dev_ptr, nbytes):
    _check(load().anakin_weight_arena_import(device, _vp(dev_ptr), nbytes), "weight_arena_import")


class Worker:
    """Worker<NV, P>: thread pool of per-thread Nets, optionally one GPU per thread."""

    def __init__(self, model_path, precision="fp32", threads=1, devices=(), batch=0):
        self._lib = load()
        self._h = _vp()
        devs = (_i * max(1, len(devices)))(*devices) if devices else None
        _check(self._lib.anakin_worker_create(model_path.encode(), PRECISIONS[precision], threads, devs,
                                              len(devices), batch, C.byref(self._h)), "Worker")

    def sync_prediction(self, x_nchw, out_count):
        a = np.ascontiguousarray(x_nchw, np.float32)
        out = np.empty(out_count, np.float32)
        _check(self._lib.anakin_worker_sync_prediction(self._h, a.ctypes.data_as(_vp), a.size,
                                                       out.ctypes.data_as(_vp), out.size), "sync_prediction")
        return out

    def wait_ready(self):
        _check(self._lib.anakin_worker_wait_ready(self._h), "Worker init")

    def async_prediction_ptr(self, in_ptr, in_count, out_ptr, out_count):
        """Queue one request on caller-owned (pinned) fp32 host buffers; pair with async_get_result()."""
        _check(self._lib.anakin_worker_async_prediction(self._h, _vp(in_ptr), in_count, _vp(out_ptr), out_count),
               "async_prediction")

    def sync_prediction_image(self, images_nhwc, out_count):
        """One request on an image input: uint8 [n, h, w, c] pixels; returns the first output (fp32)."""
        a = np.ascontiguousarray(images_nhwc)
        if a.dtype != np.uint8:
            raise AnakinError("sync_prediction_image: uint8 pixels expected, got %s" % a.dtype)
        out = np.empty(out_count, np.float32)
        _check(self._lib.anakin_worker_sync_prediction_image(self._h, a.ctypes.data_as(_vp), a.nbytes,
                                                             out.ctypes.data_as(_vp), out.size), "sync_prediction_image")
        return out

    def async_prediction_image_ptr(self, in_ptr, in_bytes, out_ptr, out_count):
        """Queue one request on caller-owned (pinned) host buffers: uint8 image bytes in, fp32 out; pair with
        async_get_result()."""
        _check(self._lib.anakin_worker_async_prediction_image(self._h, _vp(in_ptr), in_bytes, _vp(out_ptr), out_count),
               "async_prediction_image")

    def sync_prediction_images(self, images, out_count):
        """One request on an image input with on-device resize: a list of uint8 [h_i, w_i, c] arrays (the batch);
        returns the first output (fp32)."""
        pix, hw = pack_images(images)
        out = np.empty(out_count, np.float32)
        _check(self._lib.anakin_worker_sync_prediction_images(self._h, pix.ctypes.data_as(_vp), pix.nbytes,
                                                              hw.ctypes.data_as(_vp), hw.shape[0],
                                                              out.ctypes.data_as(_vp), out.size),
               "sync_prediction_images")
        return out

    def async_prediction_images_ptr(self, pix_ptr, nbytes, hw_ptr, count, out_ptr, out_count):
        """Queue one request on caller-owned (pinned) host buffers: packed uint8 pixels (pack_images), int32
        [count][2] sizes, fp32 out; all three stay the caller's until the matching async_get_result()."""
        _check(self._lib.anakin_worker_async_prediction_images(self._h, _vp(pix_ptr), nbytes, _vp(hw_ptr), count,
                                                               _vp(out_ptr), out_count), "async_prediction_images")

    def async_get_result(self):
        _check(self._lib.anakin_worker_async_get_result(self._h), "async_get_result")

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.anakin_worker_destroy(self._h)
            self._h = _vp()
