"""Host-side Python mirror of OnnxStream's FFI surface (reference: src/exports.cpp:42-311, src/bindings.py).

`Model` drives any shared library that exports the 16 ``model_*`` C entry points declared in
``include/onnxstream_b200.h`` -- the engine (``onnxstream_b200/csrc/libonnxstream_b200.so``) by default; the
test-suite points the same class at the reference compiled in place, so both sides of a parity test are driven
identically.  This module never loads a checker library on its own.  Method names,
argument meaning and error behaviour follow the reference's ``bindings.py`` so parity tests read the same on
both libraries.  No torch types cross this boundary: numpy arrays in, numpy arrays out.
"""
from __future__ import annotations

import ctypes
import os
import re
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ENGINE_LIB = os.environ.get("OSB_ENGINE_LIB") or os.path.join(_PKG_DIR, "csrc", "libonnxstream_b200.so")   # OSB_ENGINE_LIB: build variants (A/B runs)

OPTION_NAMES = (
    "use_fp16_arithmetic", "use_uint8_qdq", "use_uint8_arithmetic", "fuse_ops_in_attention",
    "force_fp16_storage", "support_dynamic_shapes", "use_ops_cache", "use_scaled_dp_attn_op",
    "use_next_op_cache", "ops_printf", "ops_times_printf", "use_nchw_convs",
)


class OnnxStreamError(RuntimeError):
    pass


class _TensorView(ctypes.Structure):  # src/exports.cpp:217-223
    _fields_ = [("dims_num", ctypes.c_size_t), ("dims", ctypes.POINTER(ctypes.c_size_t)),
                ("data_num", ctypes.c_size_t), ("data", ctypes.POINTER(ctypes.c_float))]


def mangle(name: str) -> str:
    """onnx2txt name mangling: every char outside [A-Za-z0-9] becomes _HEX_ (src/bindings.py:311-329)."""
    return re.sub(r"[^A-Za-z0-9]", lambda m: "_%02X_" % ord(m.group(0)), name)


_libs: Dict[str, ctypes.CDLL] = {}


def load_library(path: str) -> ctypes.CDLL:
    path = os.path.abspath(path)
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise OnnxStreamError(f"shared library not found: {path} (run `python -c 'import __graft_entry__ as g; g.build()'`)")
    lib = ctypes.CDLL(path)
    vp, cp, ui = ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint
    proto = {
        "model_new": ([], vp), "model_new_2": ([ctypes.c_int, cp], vp), "model_delete": ([vp], None),
        "model_read_string": ([vp, cp], None), "model_read_file": ([vp, cp], vp),
        "model_get_weights_names": ([vp], vp), "model_add_weights_file": ([vp, cp, cp, ui], vp),
        "model_add_tensor": ([vp, cp, cp, ui, ctypes.POINTER(ui)], vp), "model_get_tensor": ([vp, cp], vp),
        "model_get_all_tensor_names": ([vp], vp), "model_run": ([vp], None), "model_run_2": ([vp], vp),
        "model_clear_tensors": ([vp], None), "model_set_option": ([vp, cp, ui], None),
        "model_add_extra_output": ([vp, cp], None), "model_free_buffer": ([vp], None),
    }
    for name, (args, res) in proto.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    ext = {
        "model_ext_set_attention_parts": ([vp, ui], None), "model_ext_set_range": ([vp, cp, ctypes.c_float, ctypes.c_float], None),
        "model_ext_read_range_data": ([vp, cp], vp), "model_ext_add_upcast_pattern": ([vp, cp], None),
        "model_ext_get_tensor_i64": ([vp, cp, ctypes.POINTER(ctypes.c_longlong), ctypes.c_longlong,
                                      ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_size_t)], ctypes.c_longlong),
        "model_ext_get_tensor_type": ([vp, cp], ctypes.c_int),
        "model_ext_push_tensor": ([vp, cp, cp, ui, ctypes.POINTER(ui), vp], None),
        "model_ext_get_tensor_at": ([vp, cp, ui], vp), "model_ext_add_output_convert": ([vp, cp], None),
        "model_b200_get_stats": ([vp, ctypes.POINTER(ctypes.c_double), ctypes.c_int], ctypes.c_int),
        "model_b200_set_comm": ([vp, vp, ctypes.c_int, ctypes.c_int], ctypes.c_int),
        "model_b200_run_resident": ([vp, ctypes.c_int], ctypes.c_double),
        "model_b200_plan_summary": ([cp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int], vp),
        "osb_tc_profile": ([ctypes.c_int], None), "osb_tc_profile_read": ([ctypes.POINTER(ctypes.c_double)], ctypes.c_int),
        "osb_comm_unique_id": ([ctypes.c_char_p], ctypes.c_int), "osb_comm_init": ([ctypes.c_int, ctypes.c_int, ctypes.c_char_p], vp),
        "osb_comm_destroy": ([vp], None),
    }
    for name, (args, res) in ext.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.argtypes, fn.restype = args, res
    _libs[path] = lib
    return lib


def plan_summary(model_text: str, fp16_arithmetic: bool = True, fuse_nodes: bool = True, fuse_attention: bool = True,
                 use_scaled_dp_attn_op: bool = False, library_path: Optional[str] = None) -> str:
    """Engine only, needs no GPU: the fusion plan for `model_text` -- one line per execution step
    ("KIND n_ops first_op_type first_op_name") and a final "#summary" line (include/onnxstream_b200.h)."""
    lib = load_library(library_path or ENGINE_LIB)
    p = lib.model_b200_plan_summary(model_text.encode(), int(fp16_arithmetic), int(fuse_nodes), int(fuse_attention), int(use_scaled_dp_attn_op))
    if not p:
        raise OnnxStreamError("model_b200_plan_summary returned NULL")
    try:
        out = ctypes.string_at(p).decode()
    finally:
        lib.model_free_buffer(p)
    if out.startswith("=== ERROR ==="):
        raise OnnxStreamError(out)
    return out


class Model:
    """One OnnxStream model instance behind the C ABI."""

    def __init__(self, library_path: Optional[str] = None, threads_count: int = 0, weights_provider_name: str = "nocache",
                 plain_abi: bool = False):
        """plain_abi=True restricts the wrapper to the reference's 16 entry points (no model_ext_* / model_b200_*)."""
        self.plain_abi = plain_abi
        self.lib = load_library(library_path or ENGINE_LIB)
        self.h = self.lib.model_new_2(threads_count, weights_provider_name.encode())
        if not self.h:
            raise OnnxStreamError(f"model_new_2 failed (weights provider {weights_provider_name!r})")
        self.wp = weights_provider_name

    # -- lifetime --
    def close(self):
        if getattr(self, "h", None):
            self.lib.model_delete(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- helpers --
    def _take_string(self, ptr) -> str:
        s = ctypes.cast(ptr, ctypes.c_char_p).value.decode()
        self.lib.model_free_buffer(ptr)
        return s

    def _check(self, err_ptr):
        if err_ptr:
            raise OnnxStreamError(self._take_string(err_ptr))

    # -- model definition --
    def read_file(self, path: str):
        self._check(self.lib.model_read_file(self.h, path.encode()))

    def read_string(self, text: str):
        self.lib.model_read_string(self.h, text.encode())

    def get_weights_names(self) -> List[Tuple[str, str]]:
        s = self._take_string(self.lib.model_get_weights_names(self.h))
        return [tuple(x.split(":", 1)) for x in s.split("|")] if s else []

    def add_weights_file(self, dtype: str, name: str, data: np.ndarray):
        """'ram' provider only: copy a weight blob into engine-owned storage (src/exports.cpp:150-167)."""
        data = np.ascontiguousarray(data)
        ptr = self.lib.model_add_weights_file(self.h, dtype.encode(), name.encode(), data.nbytes)
        if not ptr:
            raise OnnxStreamError("model_add_weights_file: weights provider is not 'ram'")
        ctypes.memmove(ptr, data.ctypes.data, data.nbytes)

    # -- options --
    def set_option(self, name: str, value: bool = True):
        self.lib.model_set_option(self.h, name.encode(), 1 if value else 0)

    def add_extra_output(self, name: str):
        self.lib.model_add_extra_output(self.h, name.encode())

    # -- tensors --
    def add_tensor(self, name: str, array: np.ndarray):
        if array.dtype == np.float32:
            t = "float32"
        elif array.dtype == np.int64:
            t = "int64"
        else:
            raise OnnxStreamError("add_tensor: only float32 and int64 inputs are supported (src/exports.cpp:182-193)")
        array = np.ascontiguousarray(array)
        dims = (ctypes.c_uint * array.ndim)(*array.shape)
        if not self.plain_abi and hasattr(self.lib, "model_ext_push_tensor"):
            # Model::push_tensor semantics (works with use_fp16_arithmetic set, unlike the reference's model_add_tensor)
            self.lib.model_ext_push_tensor(self.h, t.encode(), name.encode(), array.ndim, dims, array.ctypes.data)
            return
        ptr = self.lib.model_add_tensor(self.h, t.encode(), name.encode(), array.ndim, dims)
        ctypes.memmove(ptr, array.ctypes.data, array.nbytes)

    def get_tensor(self, name: str, index: int = 0) -> Optional[np.ndarray]:
        """index > 0 (engine only): the index-th batch sibling pushed / produced under `name`."""
        ptr = self.lib.model_get_tensor(self.h, name.encode()) if index == 0 else self.lib.model_ext_get_tensor_at(self.h, name.encode(), index)
        if not ptr:
            return None
        view = ctypes.cast(ptr, ctypes.POINTER(_TensorView)).contents
        shape = tuple(view.dims[i] for i in range(view.dims_num))
        out = np.ctypeslib.as_array(view.data, shape=(view.data_num,)).copy().reshape(shape) if view.data_num else np.zeros(shape, np.float32)
        self.lib.model_free_buffer(ptr)
        return out

    def get_all_tensor_names(self) -> List[str]:
        s = self._take_string(self.lib.model_get_all_tensor_names(self.h))
        return s.split("|") if s else []

    def clear_tensors(self):
        self.lib.model_clear_tensors(self.h)

    def run(self):
        self._check(self.lib.model_run_2(self.h))

    # -- extensions (Model members the reference's apps set directly, src/onnxstream.h:944-968) --
    def set_attention_parts(self, parts: int):
        self.lib.model_ext_set_attention_parts(self.h, parts)

    def set_range(self, op_name: str, mn: float, mx: float):
        self.lib.model_ext_set_range(self.h, op_name.encode(), mn, mx)

    def read_range_data(self, path: str):
        self._check(self.lib.model_ext_read_range_data(self.h, path.encode()))

    def add_upcast_pattern(self, pattern: str):
        self.lib.model_ext_add_upcast_pattern(self.h, pattern.encode())

    def get_tensor_i64(self, name: str) -> Optional[np.ndarray]:
        cap = 1 << 20
        buf = (ctypes.c_longlong * cap)()
        dims = (ctypes.c_size_t * 8)()
        nd = ctypes.c_size_t(0)
        n = self.lib.model_ext_get_tensor_i64(self.h, name.encode(), buf, cap, dims, ctypes.byref(nd))
        if n < 0:
            return None
        return np.array(buf[:n], dtype=np.int64).reshape(tuple(dims[i] for i in range(nd.value)))

    STAT_FIELDS = ("weight_ring_bytes", "weight_peak_live_bytes", "weight_largest_node_bytes", "weight_bytes_streamed",
                   "weight_resident_bytes", "act_high_water_bytes", "h2d_input_bytes", "d2h_output_bytes", "kernel_launches",
                   "tc_launches", "steps_executed", "ops_fused_away", "last_run_ms", "last_gpu_ms", "graph_replays", "side_steps")

    def run_resident(self, steps: int) -> float:
        """Engine only: replay the captured CUDA graph `steps` times on device-resident inputs; returns CUDA-event ms."""
        ms = self.lib.model_b200_run_resident(self.h, steps)
        if ms < 0:
            raise OnnxStreamError("model_b200_run_resident failed (no captured graph?)")
        return ms

    def stats(self) -> Dict[str, float]:
        """Engine only: streaming / launch statistics of the last run (include/onnxstream_b200.h)."""
        out = (ctypes.c_double * len(self.STAT_FIELDS))()
        self.lib.model_b200_get_stats(self.h, out, len(self.STAT_FIELDS))
        return dict(zip(self.STAT_FIELDS, list(out)))
