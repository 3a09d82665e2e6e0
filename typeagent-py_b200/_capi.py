"""ctypes binding of libtavec.so (``include/tavec.h``) — the only way Python reaches the GPU.

Fails loudly: a missing library, a missing symbol or a missing CUDA device raise
``RuntimeError``; nothing here or above it computes on the CPU instead.
"""

from __future__ import annotations

import ctypes as C
import os
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libtavec.so")

TAV_F32, TAV_BF16, TAV_F16 = 0, 1, 2
DTYPE_CODES = {"float32": TAV_F32, "bfloat16": TAV_BF16, "float16": TAV_F16}
DTYPE_NAMES = {v: k for k, v in DTYPE_CODES.items()}

TAV_NORMALIZE = 1
TAV_QUERIES_ON_DEVICE, TAV_OUTPUTS_ON_DEVICE, TAV_FORCE_SCAN, TAV_FORCE_MMA, TAV_DEFER_RETRY = 1, 2, 4, 8, 16
TAV_USE_ROW_MASK, TAV_TIES_LOW_FIRST, TAV_NO_FUSED_SCAN, TAV_ITEMS_AS_POSITIONS = 32, 64, 128, 256
TAV_USE_QUERY_MASKS = 512
ABI_VERSION = 2

TAV_ERR_INVALID, TAV_ERR_CUDA, TAV_ERR_OOM, TAV_ERR_RANGE, TAV_ERR_STATE, TAV_ERR_PEER = -1, -2, -3, -4, -5, -6

# every symbol include/tavec.h declares: (name, restype, argtypes)
_i64p = C.POINTER(C.c_int64)
_f32p = C.POINTER(C.c_float)
_i32p = C.POINTER(C.c_int32)
SIGNATURES = {
    "tav_abi_version": (C.c_int, []),
    "tav_last_error": (C.c_char_p, []),
    "tav_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "tav_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_void_p)]),
    "tav_destroy": (C.c_int, [C.c_void_p]),
    "tav_clear": (C.c_int, [C.c_void_p]),
    "tav_reserve": (C.c_int, [C.c_void_p, C.c_int64]),
    "tav_append": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "tav_adopt_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int]),
    "tav_size": (C.c_int64, [C.c_void_p]),
    "tav_dim": (C.c_int, [C.c_void_p]),
    "tav_store_dtype": (C.c_int, [C.c_void_p]),
    "tav_device": (C.c_int, [C.c_void_p]),
    "tav_read_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "tav_remove_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "tav_write_rows": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int,
                                 C.c_void_p]),
    "tav_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int,
                             C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                             C.c_void_p]),
    "tav_range_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_int64,
                                   C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "tav_search_subsets": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_range_search_subsets": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_search_subsets_into": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p,
                                          C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_range_search_subsets_into": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p,
                                                C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p]),
    "tav_range_fetch": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "tav_range_search_into": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_int64,
                                        C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "tav_finish_search": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]),
    "tav_set_row_mask": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "tav_set_query_masks": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p]),
    "tav_fold_groups": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int64,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_set_row_groups": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "tav_range_search_groups": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_int64, C.c_void_p,
                                          C.c_void_p]),
    "tav_range_fetch_groups": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_void_p]),
    "tav_search_groups": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]),
    "tav_group_handle_bytes": (C.c_int, []),
    "tav_group_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "tav_group_local_handle": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tav_group_connect": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tav_group_capacity": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tav_group_destroy": (C.c_int, [C.c_void_p]),
    "tav_sharded_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int,
                                     C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_sharded_search_subset": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int,
                                            C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p]),
    "tav_sharded_finish": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]),
    "tav_group_range_reserve": (C.c_int, [C.c_void_p, C.c_int, C.c_int64]),
    "tav_group_range_handle": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tav_group_range_connect": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tav_group_range_capacity": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), _i64p]),
    "tav_sharded_range_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int,
                                           C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                           C.c_void_p, C.c_void_p]),
    "tav_sharded_range_republish": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tav_sharded_range_abort": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tav_sharded_range_merge": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_rows_handle_bytes": (C.c_int, []),
    "tav_rows_export": (C.c_int, [C.c_void_p, C.c_void_p, _i64p]),
    "tav_rows_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_rows_commit": (C.c_int, [C.c_void_p, C.c_int]),
    "tav_timing_history": (C.c_int, [C.c_void_p, C.c_int, _f32p, _f32p, _f32p, _f32p, C.POINTER(C.c_int)]),
    "tav_merge_topk": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_int64, C.c_int64, C.c_int64,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_merge_topk_ordered": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_int64, C.c_int64, C.c_int64, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_map_items": (C.c_int, [C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tav_merge_range": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                  C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_multi_create": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "tav_multi_destroy": (C.c_int, [C.c_void_p]),
    "tav_multi_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int,
                                   C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tav_multi_range_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p,
                                         C.c_int64, C.c_int64, C.c_void_p]),
    "tav_multi_range_fetch": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "tav_mma_scores": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "tav_set_timing": (C.c_int, [C.c_void_p, C.c_int]),
    "tav_timing_breakdown": (C.c_int, [C.c_void_p, _f32p, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int)]),
    "tav_last_timing": (C.c_int, [C.c_void_p, _f32p, _f32p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
}

_lib = None
_lock = threading.Lock()


def load() -> C.CDLL:
    """Load libtavec.so once and bind every declared symbol."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python typeagent-py_b200/build.py` "
                "(or __graft_entry__.build()).  There is no CPU fallback."
            )
        lib = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            try:
                fn = getattr(lib, name)
            except AttributeError as e:  # pragma: no cover - build mismatch
                raise RuntimeError(f"libtavec.so does not export {name}") from e
            fn.restype = restype
            fn.argtypes = argtypes
        if lib.tav_abi_version() != ABI_VERSION:
            raise RuntimeError(f"libtavec.so ABI version {lib.tav_abi_version()} != {ABI_VERSION}; rebuild")
        _lib = lib
    return _lib


HOST_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libtavhost.so")
_pack_int_list = False  # False = not probed yet, None = unavailable


def pack_int_list():
    """`tavhost_pack_int_list(list, int64* out, cap) -> n | -1 | -2` from libtavhost.so (csrc/tav_pyhost.c),
    or None when that optional helper was not built.  Host-side convenience only (a Python list of
    ordinals -> int64 buffer in 4 us instead of 18 us); it is not on the compute path."""
    global _pack_int_list
    if _pack_int_list is False:
        fn = None
        if os.path.exists(HOST_LIB_PATH):
            try:
                fn = C.PyDLL(HOST_LIB_PATH).tavhost_pack_int_list
                fn.restype = C.c_longlong
                fn.argtypes = [C.py_object, C.c_void_p, C.c_longlong]
            except (OSError, AttributeError):
                fn = None
        _pack_int_list = fn
    return _pack_int_list


def last_error() -> str:
    msg = load().tav_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int) -> None:
    """Map a negative tav_status to the exception the reference would raise."""
    if rc >= 0:
        return
    msg = last_error() or f"libtavec error {rc}"
    if rc == TAV_ERR_INVALID:
        raise ValueError(msg)
    if rc == TAV_ERR_RANGE:
        raise IndexError(msg)
    if rc == TAV_ERR_OOM:
        raise MemoryError(msg)
    raise RuntimeError(msg)


def device_count() -> int:
    n = C.c_int(0)
    check(load().tav_device_count(C.byref(n)))
    return n.value
