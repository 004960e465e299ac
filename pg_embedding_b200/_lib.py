"""ctypes binding of libpgemb_b200.so (the C ABI in include/pgemb_b200.h).

This is the only way Python reaches the product path; it loads the in-tree shared library built by
pg_embedding_b200/build.py and FAILS LOUDLY if it is missing -- there is no CPU or PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libpgemb_b200.so")

PGEMB_OK = 0


class HnswMetadata(C.Structure):
    """Layout-identical to the reference's HnswMetadata (embedding.h:28-42)."""
    _fields_ = [
        ("dim", C.c_size_t), ("data_size", C.c_size_t), ("offset_data", C.c_size_t),
        ("offset_label", C.c_size_t), ("size_data_per_element", C.c_size_t),
        ("elems_per_page", C.c_size_t), ("M", C.c_size_t), ("maxM", C.c_size_t),
        ("efConstruction", C.c_size_t), ("efSearch", C.c_size_t),
        ("enterpoint_node", C.c_uint32), ("dist_func", C.c_int),
    ]


class PgembHostIndex(C.Structure):
    _fields_ = [("meta", HnswMetadata), ("dev", C.c_void_p)]


# every symbol include/pgemb_b200.h declares (tests/test_abi.py checks the .so exports them all)
ABI_SYMBOLS = [
    "hnsw_search", "hnsw_bind_point", "hnsw_dist_func", "hnsw_init_dist_func", "hnsw_is_deleted",
    "pgemb_last_error", "pgemb_version", "pgemb_device_count", "pgemb_meta_init",
    "pgemb_index_create", "pgemb_index_destroy", "pgemb_index_size", "pgemb_index_capacity",
    "pgemb_index_device", "pgemb_index_append", "pgemb_index_append_device",
    "pgemb_index_append_records", "pgemb_index_export_records", "pgemb_index_get_links",
    "pgemb_index_set_links", "pgemb_index_get_labels", "pgemb_index_set_labels",
    "pgemb_index_truncate", "pgemb_index_reserve", "pgemb_search_batch", "pgemb_search_batch_device",
    "pgemb_index_poll_error", "pgemb_last_kernel_ms", "pgemb_launch_count", "pgemb_dist_batch", "pgemb_dist_gather", "pgemb_scan_topk",
    "pgemb_scan_counters", "pgemb_scan_topk_device", "pgemb_scan_topk_op", "pgemb_scan_topk_op_device", "pgemb_sharded_scan_device", "pgemb_debug_umma_product",
    "pgemb_index_scan_begin", "pgemb_index_scan_next", "pgemb_index_scan_next_batch", "pgemb_index_scan_ef", "pgemb_index_scan_searches",
    "pgemb_index_scan_end",
    "pgemb_bind_point", "pgemb_insert_batch", "pgemb_merge_topk_device", "pgemb_packed_topk_bytes", "pgemb_merge_topk_packed_device",
    "pgemb_exchange_create", "pgemb_exchange_destroy", "pgemb_exchange_handle", "pgemb_exchange_buffer", "pgemb_exchange_attach",
    "pgemb_sharded_search_device", "pgemb_sharded_merge_device", "pgemb_exchange_last_merge_ms", "pgemb_exchange_error", "pgemb_build_bulk", "pgemb_build_exact",
]

_lib = None


class PgembError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"pgemb status {status}: {msg}")
        self.status = status


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build the CUDA extension first (python -m pg_embedding_b200.build). "
            "There is no CPU fallback for the pg_embedding hot path.")
    _lib = _bind(C.CDLL(LIB_PATH))
    return _lib


def _bind(lib: C.CDLL) -> C.CDLL:
    """Attach the prototypes of include/pgemb_b200.h to a loaded library."""
    vp, sz = C.c_void_p, C.c_size_t
    f32p, u64p, u32p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)
    mp = C.POINTER(HnswMetadata)
    lib.pgemb_last_error.restype = C.c_char_p
    lib.pgemb_version.restype = C.c_char_p
    lib.pgemb_device_count.restype = C.c_int
    lib.pgemb_launch_count.restype = C.c_uint64
    lib.pgemb_meta_init.argtypes = [mp, sz, sz, sz, sz, C.c_int]
    lib.pgemb_index_create.argtypes = [mp, sz, C.c_int, C.POINTER(vp)]
    lib.pgemb_index_destroy.argtypes = [vp]
    lib.pgemb_index_destroy.restype = None
    lib.pgemb_index_size.argtypes = [vp]
    lib.pgemb_index_size.restype = sz
    lib.pgemb_index_capacity.argtypes = [vp]
    lib.pgemb_index_capacity.restype = sz
    lib.pgemb_index_device.argtypes = [vp]
    lib.pgemb_index_append.argtypes = [vp, sz, f32p, u64p, u32p]
    lib.pgemb_index_append_device.argtypes = [vp, sz, vp, vp, vp, vp]
    lib.pgemb_index_append_records.argtypes = [vp, sz, vp, sz]
    lib.pgemb_index_export_records.argtypes = [vp, sz, sz, vp, sz]
    lib.pgemb_index_get_links.argtypes = [vp, sz, sz, u32p]
    lib.pgemb_index_set_links.argtypes = [vp, sz, sz, u32p]
    lib.pgemb_index_get_labels.argtypes = [vp, sz, sz, u64p]
    lib.pgemb_index_set_labels.argtypes = [vp, sz, sz, u64p]
    lib.pgemb_index_truncate.argtypes = [vp]
    lib.pgemb_index_reserve.argtypes = [vp, sz]
    lib.pgemb_search_batch.argtypes = [vp, sz, f32p, sz, u64p, f32p, u32p, i32p, u32p]
    lib.pgemb_search_batch_device.argtypes = [vp, sz, vp, sz, vp, vp, vp, vp, vp, vp]
    lib.pgemb_index_poll_error.argtypes = [vp, vp]
    lib.pgemb_last_kernel_ms.argtypes = [vp]
    lib.pgemb_last_kernel_ms.restype = C.c_float
    lib.pgemb_dist_batch.argtypes = [C.c_int, sz, sz, f32p, C.c_int, f32p, f32p]
    lib.pgemb_dist_gather.argtypes = [vp, sz, f32p, sz, u32p, f32p]
    lib.pgemb_scan_topk.argtypes = [vp, sz, f32p, sz, u64p, f32p, i32p]
    lib.pgemb_scan_topk_op.argtypes = [vp, C.c_int, sz, f32p, sz, u64p, f32p, i32p]
    lib.pgemb_scan_counters.argtypes = [u64p]
    lib.pgemb_scan_counters.restype = None
    lib.pgemb_debug_umma_product.argtypes = [vp, sz, f32p, sz, sz, f32p]
    lib.pgemb_index_scan_begin.argtypes = [vp, f32p, sz, C.POINTER(vp)]
    lib.pgemb_index_scan_next.argtypes = [vp, u64p]
    lib.pgemb_index_scan_next.restype = C.c_int
    lib.pgemb_index_scan_next_batch.argtypes = [vp, sz, u64p, C.POINTER(sz)]
    lib.pgemb_index_scan_ef.argtypes = [vp]
    lib.pgemb_index_scan_ef.restype = sz
    lib.pgemb_index_scan_searches.argtypes = [vp]
    lib.pgemb_index_scan_searches.restype = C.c_uint64
    lib.pgemb_index_scan_end.argtypes = [vp]
    lib.pgemb_index_scan_end.restype = None
    lib.pgemb_bind_point.argtypes = [vp, C.c_uint32]
    lib.pgemb_insert_batch.argtypes = [vp, sz, f32p, u64p]
    lib.pgemb_merge_topk_device.argtypes = [sz, sz, sz, vp, vp, vp, vp, vp, vp, vp]
    lib.pgemb_packed_topk_bytes.argtypes = [sz, sz]
    lib.pgemb_packed_topk_bytes.restype = sz
    lib.pgemb_merge_topk_packed_device.argtypes = [sz, sz, sz, vp, sz, vp, vp, vp, vp]
    lib.pgemb_exchange_create.argtypes = [C.c_int, C.c_int, C.c_int, sz, sz, C.POINTER(vp)]
    lib.pgemb_exchange_destroy.argtypes = [vp]
    lib.pgemb_exchange_destroy.restype = None
    lib.pgemb_exchange_handle.argtypes = [vp, vp]
    lib.pgemb_exchange_buffer.argtypes = [vp]
    lib.pgemb_exchange_buffer.restype = vp
    lib.pgemb_exchange_attach.argtypes = [vp, vp, C.c_int]
    lib.pgemb_sharded_search_device.argtypes = [vp, vp, sz, vp, sz, vp]
    lib.pgemb_sharded_scan_device.argtypes = [vp, vp, sz, vp, sz, vp]
    lib.pgemb_scan_topk_device.argtypes = [vp, sz, vp, sz, vp, vp, vp, vp]
    lib.pgemb_scan_topk_op_device.argtypes = [vp, C.c_int, sz, vp, sz, vp, vp, vp, vp]
    lib.pgemb_sharded_merge_device.argtypes = [vp, sz, vp, vp, vp, vp]
    lib.pgemb_exchange_last_merge_ms.argtypes = [vp]
    lib.pgemb_exchange_last_merge_ms.restype = C.c_float
    lib.pgemb_exchange_error.argtypes = [vp]
    lib.pgemb_build_bulk.argtypes = [vp, sz, sz, sz, C.POINTER(C.c_double)]
    lib.pgemb_build_exact.argtypes = [vp, sz, sz, sz, C.POINTER(C.c_double), u64p]
    lib.hnsw_search.argtypes = [mp, f32p, C.POINTER(sz), C.POINTER(u64p)]
    lib.hnsw_search.restype = C.c_bool
    lib.hnsw_bind_point.argtypes = [mp, f32p, C.c_uint32]
    lib.hnsw_bind_point.restype = C.c_bool
    lib.hnsw_dist_func.argtypes = [C.c_int, f32p, f32p, sz]
    lib.hnsw_dist_func.restype = C.c_float
    lib.hnsw_init_dist_func.restype = None
    lib.hnsw_is_deleted.argtypes = [C.c_uint64]
    lib.hnsw_is_deleted.restype = C.c_bool
    return lib


def check(status: int) -> None:
    if status != PGEMB_OK:
        raise PgembError(status, load().pgemb_last_error().decode("utf-8", "replace"))
