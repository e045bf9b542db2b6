"""ctypes bindings of the two in-tree native libraries (C ABI, see ``_build.py``).

Reference: the pybind11 module ``libexb`` (openembedding/entry/py_api.cc:225-...) over the C ABI of
openembedding/entry/c_api.h; here the C ABI is called directly (ctypes releases the GIL on every call).

``core()`` -> ``libexb_core.so`` (CPU engine + checkpoint IO), ``cuda()`` ->
``libexb_cuda.so`` (sm_90a kernels). Loading is lazy; a missing/stale library is
rebuilt if a compiler is present, otherwise an ImportError explains what is missing --
on a GPU box the CUDA ops never silently fall back to eager PyTorch.
"""
import ctypes
import threading
from ctypes import (POINTER, c_char_p, c_double, c_int, c_int32, c_int64, c_uint32, c_uint64,
                    c_void_p)

from . import _build

_lock = threading.Lock()
_core = None
_cuda = None

u64p = POINTER(c_uint64)
f64p = POINTER(c_double)
i32p = POINTER(c_int32)


def _proto(lib, name, restype, argtypes):
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = argtypes
    return fn


def core():
    global _core
    if _core is not None:
        return _core
    with _lock:
        if _core is not None:
            return _core
        path = _build.build_core()
        lib = ctypes.CDLL(path)
        P = _proto
        P(lib, "exb_core_version", c_char_p, [])
        P(lib, "exb_var_create", c_void_p, [c_int, c_int, c_uint64, c_int, c_int, c_int])
        P(lib, "exb_var_destroy", None, [c_void_p])
        P(lib, "exb_var_set_initializer", None, [c_void_p, c_int, c_double, c_double, c_double, c_uint64])
        P(lib, "exb_var_set_optimizer", None, [c_void_p, c_int, f64p, c_int])
        P(lib, "exb_var_state_dim", c_int, [c_void_p])
        P(lib, "exb_var_pull", None, [c_void_p, c_void_p, c_uint64, c_void_p])
        P(lib, "exb_var_push", None, [c_void_p, c_void_p, c_uint64, c_void_p, c_void_p])
        P(lib, "exb_var_update", None, [c_void_p])
        P(lib, "exb_var_pending", c_uint64, [c_void_p])
        P(lib, "exb_var_num_items", c_uint64, [c_void_p])
        P(lib, "exb_var_read_indices", c_uint64, [c_void_p, u64p, c_void_p, c_uint64])
        P(lib, "exb_var_get_weights", None, [c_void_p, c_void_p, c_uint64, c_void_p, c_void_p])
        P(lib, "exb_var_set_weights", None, [c_void_p, c_void_p, c_uint64, c_void_p, c_void_p, c_uint64])
        P(lib, "exb_var_clear", None, [c_void_p])
        P(lib, "exb_opt_update_rows_f32", None, [c_int, f64p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_uint64])
        P(lib, "exb_opt_update_rows_f64", None, [c_int, f64p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_uint64])
        P(lib, "exb_opt_init_state_f32", None, [c_int, f64p, c_void_p, c_int, c_uint64])
        P(lib, "exb_opt_state_dim", c_int, [c_int, c_int])
        P(lib, "exb_init_rows_f32", None, [c_int, c_double, c_double, c_double, c_uint64, c_void_p, c_uint64, c_int, c_void_p])
        P(lib, "exb_init_rows_f64", None, [c_int, c_double, c_double, c_double, c_uint64, c_void_p, c_uint64, c_int, c_void_p])
        P(lib, "exb_hash64_c", c_uint64, [c_uint64])
        P(lib, "exb_fw_open", c_void_p, [c_char_p])
        P(lib, "exb_fw_header", None, [c_void_p, c_uint32, c_int32, c_uint64, c_uint64, c_char_p, c_uint64,
                                      c_int32, c_int32, c_uint64, c_uint64])
        P(lib, "exb_fw_block", None, [c_void_p, c_uint64, c_void_p, c_void_p, c_uint64, c_void_p, c_uint64])
        P(lib, "exb_fw_close", None, [c_void_p])
        P(lib, "exb_fr_open", c_void_p, [c_char_p])
        P(lib, "exb_fr_header", c_int, [c_void_p, POINTER(c_uint32), i32p, u64p, u64p, c_char_p, c_uint64, u64p,
                                       i32p, i32p, u64p, u64p])
        P(lib, "exb_fr_block_size", c_int64, [c_void_p])
        P(lib, "exb_fr_block", c_int, [c_void_p, c_uint64, c_void_p, c_void_p, c_uint64, c_void_p, c_uint64])
        P(lib, "exb_fr_skip_block", c_int, [c_void_p, c_uint64, c_uint64, c_uint64])
        P(lib, "exb_lz4_bound", c_int64, [c_int64])
        P(lib, "exb_lz4_compress", c_int64, [c_char_p, c_int64, c_void_p, c_int64])
        P(lib, "exb_lz4_decompress", c_int64, [c_char_p, c_int64, c_void_p, c_int64])
        P(lib, "exb_fr_close", None, [c_void_p])
        P(lib, "exb_unique_indices", c_uint64, [c_void_p, c_uint64, c_void_p, c_void_p])
        _core = lib
    return _core


def cuda():
    global _cuda
    if _cuda is not None:
        return _cuda
    with _lock:
        if _cuda is not None:
            return _cuda
        path = _build.build_cuda()
        lib = ctypes.CDLL(path)
        P = _proto
        P(lib, "exb_cuda_last_error", c_char_p, [])
        P(lib, "exb_cuda_device_count", c_int, [])
        P(lib, "exb_engine_create", c_void_p, [c_int, c_int, c_int])
        P(lib, "exb_engine_destroy", None, [c_void_p])
        P(lib, "exb_engine_sms", c_int, [c_void_p])
        P(lib, "exb_engine_set_max_ctas", None, [c_void_p, c_int])
        P(lib, "exb_engine_sync_ptr", c_uint64, [c_void_p])
        P(lib, "exb_engine_sync_bytes", c_uint64, [])
        P(lib, "exb_engine_set_peer_sync", None, [c_void_p, c_int, c_uint64])
        P(lib, "exb_engine_status", c_int, [c_void_p, i32p, u64p])
        P(lib, "exb_engine_reset_status", c_int, [c_void_p])
        P(lib, "exb_table_add", c_int, [c_void_p, c_int, c_int, c_uint64, c_uint64, c_int, c_int])
        P(lib, "exb_table_set_initializer", c_int, [c_void_p, c_int, c_int, c_double, c_double, c_double, c_uint64])
        P(lib, "exb_table_set_optimizer", c_int, [c_void_p, c_int, c_int, f64p, c_int])
        P(lib, "exb_table_alloc", c_int, [c_void_p, c_int])
        P(lib, "exb_table_info", c_int, [c_void_p, c_int, u64p])
        P(lib, "exb_table_set_peer", c_int, [c_void_p, c_int, c_int, c_uint64, c_uint64])
        P(lib, "exb_engine_commit", c_int, [c_void_p])
        P(lib, "exb_engine_accept_ctx", c_int, [c_void_p])
        P(lib, "exb_engine_ctx_version", c_uint32, [c_void_p])
        P(lib, "exb_table_size", c_int, [c_void_p, c_int, u64p])
        P(lib, "exb_table_enumerate", c_int, [c_void_p, c_int, c_uint64, c_uint64, u64p, c_uint64])
        P(lib, "exb_table_gather", c_int, [c_void_p, c_int, c_uint64, c_uint64, c_uint64, c_uint64, c_uint64])
        P(lib, "exb_table_scatter", c_int, [c_void_p, c_int, c_uint64, c_uint64, c_uint64, c_uint64, c_uint64])
        P(lib, "exb_table_clear", c_int, [c_void_p, c_int])
        P(lib, "exb_table_rehash", c_int, [c_void_p, c_int, c_uint64])
        P(lib, "exb_raw_alloc", c_uint64, [c_int, c_uint64])
        P(lib, "exb_raw_free", c_int, [c_uint64])
        P(lib, "exb_ipc_get_handle", c_int, [c_uint64, c_char_p])
        P(lib, "exb_ipc_open_handle", c_uint64, [c_char_p])
        P(lib, "exb_ipc_close_handle", c_int, [c_uint64])
        P(lib, "exb_enable_peer_access", c_int, [c_int, c_int])
        P(lib, "exb_plan_create", c_void_p, [c_void_p, c_int, i32p, i32p, i32p, c_int, c_int, c_int])
        P(lib, "exb_plan_create2", c_void_p, [c_void_p, c_int, i32p, i32p, i32p, c_int, c_int, c_int, i32p, i32p])
        P(lib, "exb_plan_destroy", None, [c_void_p])
        P(lib, "exb_plan_inbox_info", c_int, [c_void_p, u64p])
        P(lib, "exb_plan_set_peer_inbox", c_int, [c_void_p, c_int, c_uint64])
        P(lib, "exb_plan_commit", c_int, [c_void_p])
        P(lib, "exb_plan_grid", c_int, [c_void_p, c_int])
        P(lib, "exb_plan_set_trace", c_int, [c_void_p, c_uint64])
        P(lib, "exb_pull", c_int, [c_void_p, c_uint64, c_uint64, c_int, c_uint64])
        P(lib, "exb_push_update", c_int, [c_void_p, c_uint64, c_uint64, c_int, c_uint64])
        P(lib, "exb_plan_prepare", c_int, [c_void_p, c_uint64, c_int, c_int, c_uint64])
        P(lib, "exb_plan_reset", c_int, [c_void_p, c_int, c_uint64])
        P(lib, "exb_pull2", c_int, [c_void_p, c_uint64, c_uint64, c_int, c_int, c_uint64])
        P(lib, "exb_push2", c_int, [c_void_p, c_uint64, c_int, c_int, c_uint64])
        P(lib, "exb_plan_set_dense_reduce", c_int, [c_void_p, ctypes.POINTER(c_uint64), c_uint64])
        P(lib, "exb_pull_plan", c_int, [c_void_p, c_uint64, c_uint64, c_int, c_int, c_uint64])
        P(lib, "exb_plan_memory", c_int, [c_void_p, u64p])
        P(lib, "exb_engine_status_ptr", c_uint64, [c_void_p])
        P(lib, "exb_ds_last_error", c_char_p, [])
        P(lib, "exb_ds_create", c_void_p, [c_int, c_int, c_int, c_uint64, c_int, c_int, c_int, c_uint64])
        P(lib, "exb_ds_destroy", None, [c_void_p])
        P(lib, "exb_ds_set_initializer", c_int, [c_void_p, c_int, c_double, c_double, c_double, c_uint64])
        P(lib, "exb_ds_set_optimizer", c_int, [c_void_p, c_int, f64p, c_int])
        P(lib, "exb_ds_state_dim", c_int, [c_void_p])
        P(lib, "exb_ds_num_items", c_uint64, [c_void_p])
        P(lib, "exb_ds_pull", c_int, [c_void_p, c_uint64, c_uint64, c_uint64, c_uint64])
        P(lib, "exb_ds_update", c_int, [c_void_p, c_uint64, c_uint64, c_uint64, c_uint64, c_uint64])
        P(lib, "exb_ds_get", c_int, [c_void_p, c_uint64, c_uint64, c_uint64, c_uint64, c_uint64])
        P(lib, "exb_ds_set", c_int, [c_void_p, c_uint64, c_uint64, c_uint64, c_uint64, c_uint64])
        P(lib, "exb_ds_enumerate", c_int, [c_void_p, c_uint64, u64p])
        P(lib, "exb_ds_clear", c_int, [c_void_p])
        P(lib, "exb_ds_status", c_int, [c_void_p])
        P(lib, "exb_ds_bytes", c_uint64, [c_void_p])
        P(lib, "exb_tier_create", c_void_p, [c_void_p, c_int, c_uint64])
        P(lib, "exb_tier_destroy", None, [c_void_p])
        P(lib, "exb_tier_admit", c_int, [c_void_p, c_uint64, c_uint64, c_uint32, c_uint64])
        P(lib, "exb_tier_flush", c_int, [c_void_p, c_uint32, c_uint64])
        P(lib, "exb_tier_evict", c_int, [c_void_p, c_uint64, c_uint32, c_uint64])
        P(lib, "exb_tier_clear", c_int, [c_void_p, c_int])
        P(lib, "exb_tier_stats", c_int, [c_void_p, u64p])
        P(lib, "exb_tier_info", c_int, [c_void_p, u64p])
        P(lib, "exb_tier_host_enumerate", c_int, [c_void_p, c_uint64, c_uint64, u64p])
        P(lib, "exb_tier_hkeys_ptr", c_uint64, [c_void_p])
        P(lib, "exb_tier_host_put", c_int, [c_void_p, c_void_p, c_uint64, c_void_p])
        P(lib, "exb_tier_relayout", c_int, [c_void_p])
        _cuda = lib
    return _cuda


def cuda_loaded():
    return _cuda is not None


def cuda_check(rc, what=""):
    if rc != 0:
        raise RuntimeError("libexb_cuda %s failed: %s" % (what, cuda().exb_cuda_last_error().decode()))
