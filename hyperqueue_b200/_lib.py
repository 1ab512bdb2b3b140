"""ctypes binding of include/hqsched.h (the same C ABI a Rust/bindgen shim would bind, INTEGRATION.md)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HQS_MAX_RESOURCES = 16
HQS_MAX_VARIANTS = 8
HQS_MAX_WORKERS = 1024
HQS_MAX_CLASSES = 4096
HQS_MAX_GROUPS = 8192
HQS_AMOUNT_MAX = (1 << 64) - 1
HQS_TIME_INF = (1 << 64) - 1
HQS_CREATE_NO_PACK, HQS_CREATE_WIDE_AMOUNTS, HQS_CREATE_SHARE_DEVICE = 1, 2, 4

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libhqsched_b200.so")

# every symbol include/hqsched.h declares
ABI_SYMBOLS = [
    "hqs_abi_version", "hqs_create", "hqs_destroy", "hqs_last_error", "hqs_classes_set", "hqs_ready_push",
    "hqs_ready_remove", "hqs_dag_load", "hqs_tasks_finished", "hqs_tick", "hqs_tick_launch", "hqs_tick_fetch",
    "hqs_shard_count", "hqs_shard_solve_emit", "hqs_device_result", "hqs_ready_rearm", "hqs_stream", "hqs_sync",
    "hqs_get_stats", "hqs_set_stream", "hqs_set_profile", "hqs_get_kernel_ms", "hqs_debug_read", "hqs_levels_add", "hqs_query",
    "hqs_shard_xbuf", "hqs_ipc_open", "hqs_shard_attach", "hqs_shard_tick_launch", "hqs_tick_reserve",
    "hqs_prefill_config", "hqs_prefill_state", "hqs_prefill_dispose", "hqs_ready_push_range", "hqs_debug_keys",
    "hqs_query_fetch", "hqs_shard_query_launch", "hqs_shard_query_solve",
    "hqs_tick_fetch_grouped", "hqs_tick_grouped", "hqs_grouped_reserve", "hqs_grouped_kernel_ms",
]
HQS_IPC_HANDLE_BYTES = 64


class LibraryNotBuilt(RuntimeError):
    pass


class HqsError(RuntimeError):
    def __init__(self, code: int, message: str) -> None:
        super().__init__(f"hqsched error {code}: {message}")
        self.code = code


class hqs_variant(C.Structure):
    _fields_ = [("amount", C.c_uint64 * HQS_MAX_RESOURCES), ("all_mask", C.c_uint32), ("weight", C.c_uint32),
                ("min_time_ms", C.c_uint64)]


class hqs_class(C.Structure):
    _fields_ = [("n_variants", C.c_uint32), ("n_nodes", C.c_uint32), ("variants", hqs_variant * HQS_MAX_VARIANTS)]


class hqs_worker(C.Structure):
    _fields_ = [("worker_id", C.c_uint32), ("flags", C.c_uint32), ("remaining_time_ms", C.c_uint64),
                ("min_utilization", C.c_float), ("reserved", C.c_uint32)]


class hqs_stats(C.Structure):
    _fields_ = [("n_groups", C.c_uint32), ("n_levels", C.c_uint32), ("n_assigned", C.c_uint32),
                ("n_segments", C.c_uint32), ("kernel_launches", C.c_uint64), ("ticks", C.c_uint64),
                ("n_handles", C.c_uint32), ("coarsened", C.c_uint32),
                ("narrow_amounts", C.c_uint32), ("solver_path", C.c_uint32)]


# hqs_stats.solver_path bits (include/hqsched.h)
HQS_PATH_WIDE, HQS_PATH_LEAN, HQS_PATH_LEAN_EXTRAS, HQS_PATH_GENERAL = 0x01, 0x02, 0x04, 0x08
HQS_PATH_PACKED, HQS_PATH_MU_RESTART, HQS_PATH_CLASSES_GLOBAL, HQS_PATH_REM_GLOBAL = 0x10, 0x20, 0x40, 0x80
HQS_PATH_EMIT_STAGED = 0x100


worker_dtype = np.dtype([("worker_id", "<u4"), ("flags", "<u4"), ("remaining_time_ms", "<u8"),
                         ("min_utilization", "<f4"), ("reserved", "<u4")])
assignment_dtype = np.dtype([("task", "<u4"), ("worker", "<u2"), ("variant", "u1"), ("kind", "u1")])
assert worker_dtype.itemsize == C.sizeof(hqs_worker) == 24
assert assignment_dtype.itemsize == 8

_lib = None
_shim = None
SHIM_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libhqtako_shim.so")


def load_shim() -> C.CDLL:
    """Loads libhqtako_shim.so, the C++ host side above the C ABI (include/tako_shim.hpp).  Python only calls its
    extern "C" self-test; C++ hosts link the library and use tako_b200::GpuCore directly."""
    global _shim
    if _shim is None:
        load_library()
        if not os.path.exists(SHIM_PATH):
            raise LibraryNotBuilt(f"{SHIM_PATH} is missing: run `python __graft_entry__.py`")
        _shim = C.CDLL(SHIM_PATH)
        _shim.hqshim_selftest.argtypes = [C.c_int, C.c_int]
        _shim.hqshim_selftest.restype = C.c_int
        _shim.hqshim_selftest_grouped.argtypes = [C.c_int, C.c_int]
        _shim.hqshim_selftest_grouped.restype = C.c_int
        _shim.hqshim_time_mapping.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int,
                                              C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64)]
        _shim.hqshim_time_mapping.restype = C.c_int
    return _shim


def load_library() -> C.CDLL:
    """Loads libhqsched_b200.so (built in-tree by __graft_entry__.build()).  No fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryNotBuilt(f"{LIB_PATH} is missing: run `python __graft_entry__.py` (nvcc, sm_90a). "
                              "hyperqueue_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, u32, u64p, u32p, u8p = C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p
    lib.hqs_abi_version.restype = C.c_int
    lib.hqs_create.argtypes = [C.POINTER(vp), C.c_int, u32, u32]
    lib.hqs_destroy.argtypes = [vp]
    lib.hqs_destroy.restype = None
    lib.hqs_last_error.argtypes = [vp]
    lib.hqs_last_error.restype = C.c_char_p
    lib.hqs_classes_set.argtypes = [vp, u32, C.POINTER(hqs_class)]
    lib.hqs_ready_push.argtypes = [vp, u32, u32p, u32p, u64p]
    lib.hqs_ready_remove.argtypes = [vp, u32, u32p]
    lib.hqs_ready_push_range.argtypes = [vp, u32, u32, u32p, u64p]
    lib.hqs_dag_load.argtypes = [vp, u32, u32p, u64p, u32p, u32p, u32p]
    lib.hqs_tasks_finished.argtypes = [vp, u32, u32p, C.POINTER(C.c_uint32)]
    lib.hqs_tick.argtypes = [vp, u32, vp, u64p, u64p, u8p, u32, vp, C.POINTER(C.c_uint32), u64p]
    lib.hqs_tick_launch.argtypes = [vp, u32, vp, u64p, u64p, u8p, u32]
    lib.hqs_tick_fetch.argtypes = [vp, u32, vp, C.POINTER(C.c_uint32), u64p]
    lib.hqs_tick_fetch_grouped.argtypes = [vp, u32, vp, C.POINTER(C.c_uint32), u32, u32p, u64p]
    lib.hqs_tick_grouped.argtypes = [vp, u32, vp, u64p, u64p, u8p, u32, vp, C.POINTER(C.c_uint32), u32, u32p, u64p]
    lib.hqs_grouped_reserve.argtypes = [vp, u32, u32]
    lib.hqs_grouped_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
    lib.hqs_shard_count.argtypes = [vp, u32, vp, u64p, u64p, u8p, vp, u32, C.POINTER(C.c_uint32)]
    lib.hqs_shard_solve_emit.argtypes = [vp, vp, vp, u32]
    lib.hqs_tick_reserve.argtypes = [vp, u32, u32, C.c_int]
    lib.hqs_shard_xbuf.argtypes = [vp, C.POINTER(vp), vp]
    lib.hqs_ipc_open.argtypes = [vp, vp, C.POINTER(vp)]
    lib.hqs_shard_attach.argtypes = [vp, u32, u32, C.POINTER(vp)]
    lib.hqs_shard_tick_launch.argtypes = [vp, u32, vp, u64p, u64p, u8p, u32]
    lib.hqs_device_result.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]
    lib.hqs_ready_rearm.argtypes = [vp]
    lib.hqs_stream.argtypes = [vp]
    lib.hqs_stream.restype = vp
    lib.hqs_sync.argtypes = [vp]
    lib.hqs_get_stats.argtypes = [vp, C.POINTER(hqs_stats)]
    lib.hqs_set_stream.argtypes = [vp, vp]
    lib.hqs_set_profile.argtypes = [vp, C.c_int]
    lib.hqs_get_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
    lib.hqs_debug_read.argtypes = [vp, C.POINTER(C.c_uint64)]
    lib.hqs_debug_keys.argtypes = [vp, u32, u32p, C.POINTER(C.c_uint32)]
    lib.hqs_levels_add.argtypes = [vp, u32, u64p]
    lib.hqs_query.argtypes = [vp, u32, vp, u64p, u64p, u8p, C.POINTER(C.c_uint32), u32p, u64p]
    lib.hqs_query_fetch.argtypes = [vp, C.POINTER(C.c_uint32), u32p, u64p]
    lib.hqs_shard_query_launch.argtypes = [vp, u32, vp, u64p, u64p, u8p]
    lib.hqs_shard_query_solve.argtypes = [vp, vp]
    lib.hqs_prefill_config.argtypes = [vp, u32, u32]
    lib.hqs_prefill_state.argtypes = [vp, u32, u8p]
    lib.hqs_prefill_dispose.argtypes = [vp, u32]
    for name in ABI_SYMBOLS:
        fn = getattr(lib, name)
        if fn.restype is C.c_int or name in ("hqs_abi_version",):
            fn.restype = C.c_int
    if lib.hqs_abi_version() != 1:
        raise RuntimeError("hqsched ABI version mismatch")
    _lib = lib
    return lib


def ptr(a: np.ndarray):
    return None if a is None else a.ctypes.data_as(C.c_void_p)
