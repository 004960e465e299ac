"""ctypes binding of libpgemb_client.so (include/pgemb_client.h) + a helper that runs a pgemb_sidecar process.

The sidecar is the one GPU-owning process of a forked-backend deployment (DESIGN.md section 12, INTEGRATION.md): it keeps
the HBM mirror of every hnsw relation and gathers the one-query-per-call `hnsw_search` requests of concurrently running
backends into batched traversal launches, their index-less scans into batched brute-force scans and their `hnsw_dist_func`
calls into batched distance launches.  This module is what tests/test_sidecar*.py and tools/bench_sidecar.py use; it
contains no computation and no fallback -- without a serving sidecar every call fails.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import time

import numpy as np

from ._lib import HnswMetadata

HERE = os.path.dirname(os.path.abspath(__file__))
CLIENT_PATH = os.path.join(HERE, "libpgemb_client.so")
SERVER_PATH = os.path.join(HERE, "pgemb_sidecar")
METRICS = {"l2": 0, "cosine": 1, "manhattan": 2}


class PgembClientIndex(C.Structure):
    """Layout of PgembClientIndex (pgemb_client.h): the reference's metadata first, then the relation key."""
    _fields_ = [("meta", HnswMetadata), ("rel_key", C.c_uint64)]


class SidecarError(RuntimeError):
    pass


_client = None


def client() -> C.CDLL:
    global _client
    if _client is not None:
        return _client
    if not os.path.isfile(CLIENT_PATH):
        raise ImportError(f"{CLIENT_PATH} is missing: python -m pg_embedding_b200.build")
    lib = C.CDLL(CLIENT_PATH)
    sz, vp = C.c_size_t, C.c_void_p
    hp = C.POINTER(PgembClientIndex)
    lib.pgemb_client_connect.argtypes = [C.c_char_p, C.c_int]
    lib.pgemb_client_last_error.restype = C.c_char_p
    lib.pgemb_client_segment_name.restype = C.c_char_p
    lib.pgemb_client_replicas.restype = C.c_int
    lib.pgemb_client_attach.argtypes = [hp, sz, C.POINTER(sz), C.POINTER(sz)]
    lib.pgemb_client_append_records.argtypes = [hp, sz, vp, sz]
    lib.pgemb_client_export_records.argtypes = [hp, sz, sz, vp, sz]
    lib.pgemb_client_get_links.argtypes = [hp, sz, sz, vp]
    lib.pgemb_client_set_labels.argtypes = [hp, sz, sz, vp]
    lib.pgemb_client_size.argtypes = [hp, C.POINTER(sz), C.POINTER(sz)]
    lib.pgemb_client_truncate.argtypes = [hp]
    lib.pgemb_client_drop.argtypes = [hp]
    lib.pgemb_client_build.argtypes = [hp, sz, sz, sz, C.c_int, C.POINTER(C.c_double)]
    lib.pgemb_client_stats.argtypes = [C.POINTER(C.c_uint64)] * 3
    lib.pgemb_client_scan_stats.argtypes = [C.POINTER(C.c_uint64)] * 3
    lib.pgemb_client_dist_stats.argtypes = [C.POINTER(C.c_uint64)] * 3
    lib.pgemb_client_scan_topk.argtypes = [hp, C.POINTER(C.c_float), sz, C.POINTER(C.c_uint64), C.POINTER(C.c_float), C.POINTER(sz)]
    lib.pgemb_client_set_interrupt_check.argtypes = [C.c_void_p]
    lib.hnsw_search.argtypes = [C.POINTER(HnswMetadata), C.POINTER(C.c_float), C.POINTER(sz), C.POINTER(C.POINTER(C.c_uint64))]
    lib.hnsw_search.restype = C.c_bool
    lib.hnsw_bind_point.argtypes = [C.POINTER(HnswMetadata), C.POINTER(C.c_float), C.c_uint32]
    lib.hnsw_bind_point.restype = C.c_bool
    lib.hnsw_dist_func.argtypes = [C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), sz]
    lib.hnsw_dist_func.restype = C.c_float
    lib.hnsw_is_deleted.argtypes = [C.c_uint64]
    lib.hnsw_is_deleted.restype = C.c_bool
    _client = lib
    return lib


_libc = C.CDLL(None)
_libc.free.argtypes = [C.c_void_p]


def _check(rc: int) -> None:
    if rc != 0:
        raise SidecarError(f"pgemb status {rc}: {client().pgemb_client_last_error().decode('utf-8', 'replace')}")


def connect(shm_name: str, timeout_ms: int = 10000) -> None:
    _check(client().pgemb_client_connect(shm_name.encode(), timeout_ms))


def stats() -> dict:
    a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
    _check(client().pgemb_client_stats(C.byref(a), C.byref(b), C.byref(c)))
    return {"batches": a.value, "searches": b.value, "max_batch": c.value}


def scan_stats() -> dict:
    """The sidecar's scan counters: pgemb_scan_topk calls, scans served, largest scan batch (not part of stats())."""
    a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
    _check(client().pgemb_client_scan_stats(C.byref(a), C.byref(b), C.byref(c)))
    return {"calls": a.value, "scans": b.value, "max_batch": c.value}


def dist_stats() -> dict:
    """The sidecar's distance counters: pgemb_dist_batch calls, hnsw_dist_func pairs served, largest distance batch (not
    part of stats() or scan_stats())."""
    a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
    _check(client().pgemb_client_dist_stats(C.byref(a), C.byref(b), C.byref(c)))
    return {"calls": a.value, "dists": b.value, "max_batch": c.value}


class RemoteIndex:
    """A backend's view of one relation's device mirror: the reference-shaped calls of embedding.h over the sidecar."""

    def __init__(self, rel_key: int, dims: int, m: int, efconstruction: int, efsearch: int, metric: str, capacity: int):
        self.h = PgembClientIndex()
        # the derived record geometry as hnsw_get_index computes it in the backend (embedding.c:222-235); a backend does
        # not load the CUDA library, so neither does this mirror of it
        if dims < 1:
            raise ValueError("HNSW index requires 'dims' to be specified")  # embedding.c:219-221
        mt = self.h.meta
        mt.dim, mt.M, mt.maxM = dims, m, 2 * m
        mt.data_size = dims * 4
        mt.offset_data = (mt.maxM + 1) * 4
        mt.offset_label = mt.offset_data + mt.data_size
        mt.size_data_per_element = mt.offset_label + 8
        mt.elems_per_page = (8192 - 24 - 4) // (mt.size_data_per_element + 4)  # BLCKSZ, page header, HnswPageOpaque, ItemIdData
        mt.efConstruction, mt.efSearch, mt.enterpoint_node, mt.dist_func = efconstruction, efsearch, 0, METRICS[metric]
        if mt.elems_per_page == 0:
            raise ValueError("Element doesn't fit in Postgres page")  # embedding.c:229-231
        self.h.rel_key = rel_key
        self.dims = dims
        size, cap = C.c_size_t(), C.c_size_t()
        _check(client().pgemb_client_attach(C.byref(self.h), capacity, C.byref(size), C.byref(cap)))
        self.capacity = cap.value

    @property
    def record_bytes(self) -> int:
        return int(self.h.meta.size_data_per_element)

    def __len__(self) -> int:
        size = C.c_size_t()
        _check(client().pgemb_client_size(C.byref(self.h), C.byref(size), None))
        return size.value

    def append_records(self, records: np.ndarray) -> None:
        r = np.ascontiguousarray(records, dtype=np.uint8)
        _check(client().pgemb_client_append_records(C.byref(self.h), r.shape[0], r.ctypes.data_as(C.c_void_p), r.shape[1]))

    def export_records(self, first: int, n: int) -> np.ndarray:
        out = np.zeros((n, self.record_bytes), np.uint8)
        _check(client().pgemb_client_export_records(C.byref(self.h), first, n, out.ctypes.data_as(C.c_void_p), out.shape[1]))
        return out

    def links(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = len(self) - first if n is None else n
        out = np.zeros((n, int(self.h.meta.maxM) + 1), np.uint32)
        _check(client().pgemb_client_get_links(C.byref(self.h), first, n, out.ctypes.data_as(C.c_void_p)))
        return out

    def set_labels(self, first: int, labels: np.ndarray) -> None:
        l = np.ascontiguousarray(labels, dtype=np.uint64)
        _check(client().pgemb_client_set_labels(C.byref(self.h), first, l.size, l.ctypes.data_as(C.c_void_p)))

    def build(self, first: int, n: int, batch_max: int = 256, exact: bool = True) -> float:
        sec = C.c_double()
        _check(client().pgemb_client_build(C.byref(self.h), first, n, batch_max, 1 if exact else 0, C.byref(sec)))
        return sec.value

    def truncate(self) -> None:
        _check(client().pgemb_client_truncate(C.byref(self.h)))

    def drop(self) -> None:
        _check(client().pgemb_client_drop(C.byref(self.h)))

    # ---- the reference-shaped calls (embedding.h:46-47) ----
    def search(self, q: np.ndarray, efsearch: int | None = None) -> np.ndarray:
        q = np.ascontiguousarray(q, dtype=np.float32)
        if q.size != self.dims:
            raise ValueError(f"Wrong number of dimensions: {q.size} instead of {self.dims} expected")  # embedding.c:311-315
        if efsearch is not None:
            self.h.meta.efSearch = efsearch
        n, res = C.c_size_t(), C.POINTER(C.c_uint64)()
        ok = client().hnsw_search(C.byref(self.h.meta), q.ctypes.data_as(C.POINTER(C.c_float)), C.byref(n), C.byref(res))
        if not ok:
            raise SidecarError("HNSW index search failed: " + client().pgemb_client_last_error().decode("utf-8", "replace"))  # embedding.c:318
        out = np.ctypeslib.as_array(res, shape=(n.value,)).copy() if n.value else np.zeros(0, np.uint64)
        _libc.free(res)  # embedding.c:327
        return out

    def scan(self, q: np.ndarray, limit: int | None = None):
        """hnsw_gettuple's iteration (embedding.c:285-370) over the reference-shaped hnsw_search of the client library: when
        the current results are used up and the search was full (n == efSearch), double efSearch in place (:334), search
        again and continue with the labels not returned before; stop when a search finds nothing new."""
        qv = np.ascontiguousarray(q, dtype=np.float32).ravel()
        ef0 = int(self.h.meta.efSearch)
        try:
            results = self.search(qv).tolist()
            returned = 0
            no_more = len(results) < int(self.h.meta.efSearch)
            while limit is None or returned < limit:
                if returned >= len(results):
                    if no_more:
                        return
                    self.h.meta.efSearch = int(self.h.meta.efSearch) * 2
                    new = self.search(qv).tolist()
                    if len(new) <= len(results):
                        return
                    no_more = len(new) < int(self.h.meta.efSearch)
                    seen = set(results)
                    results += [l for l in new if l not in seen]
                    if returned >= len(results):
                        return
                yield results[returned]
                returned += 1
        finally:
            self.h.meta.efSearch = ef0      # the reference's HnswIndex is per scan (embedding.c:254)

    def scan_topk(self, q: np.ndarray, k: int) -> dict:
        """`ORDER BY val <op> q LIMIT k` without the index (knn.out:63-91) for one query, through the sidecar's batched
        pgemb_scan_topk.  Returns dict(labels[k], dists[k], n) -- one row of HnswIndex.scan_topk (unused tail: ~0 / inf)."""
        q = np.ascontiguousarray(q, dtype=np.float32).ravel()
        if q.size != self.dims:
            raise ValueError(f"Wrong number of dimensions: {q.size} instead of {self.dims} expected")
        labels = np.full(max(int(k), 1), np.iinfo(np.uint64).max, np.uint64)
        dists = np.full(max(int(k), 1), np.inf, np.float32)
        n = C.c_size_t()
        _check(client().pgemb_client_scan_topk(C.byref(self.h), q.ctypes.data_as(C.POINTER(C.c_float)), int(k),
                                               labels.ctypes.data_as(C.POINTER(C.c_uint64)), dists.ctypes.data_as(C.POINTER(C.c_float)), C.byref(n)))
        return {"labels": labels, "dists": dists, "n": n.value}

    def bind_point(self, idx: int, efconstruction: int | None = None) -> None:
        if efconstruction is not None:
            self.h.meta.efConstruction = efconstruction
        if not client().hnsw_bind_point(C.byref(self.h.meta), None, idx):
            raise SidecarError("HNSW index insert failed: " + client().pgemb_client_last_error().decode("utf-8", "replace"))  # embedding.c:187


def dist(metric: str, a: np.ndarray, b: np.ndarray) -> np.float32:
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    f32p = C.POINTER(C.c_float)
    return np.float32(client().hnsw_dist_func(METRICS[metric], a.ctypes.data_as(f32p), b.ctypes.data_as(f32p), a.size))


class SidecarProcess:
    """Runs pgemb_sidecar as a child process (tests, benches).  `lib` = the C-ABI library it should dlopen()."""

    def __init__(self, shm_name: str, lib: str | None = None, slots: int = 64, max_dim: int = 2000, max_ef: int = 1024, bulk_mb: int = 16,
                 linger_us: int | None = None, device: int = 0, env: dict | None = None, max_batch: int | None = None):
        if not os.path.isfile(SERVER_PATH):
            raise ImportError(f"{SERVER_PATH} is missing: python -m pg_embedding_b200.build")
        self.shm_name = shm_name
        cmd = [SERVER_PATH, "--shm", shm_name, "--slots", str(slots), "--max-dim", str(max_dim), "--max-ef", str(max_ef), "--bulk-mb", str(bulk_mb),
               "--device", str(device)]
        if linger_us is not None:       # else the sidecar's default (adaptive wait of at most 50 us / a quarter of a round)
            cmd += ["--linger-us", str(linger_us)]
        if max_batch is not None:
            cmd += ["--max-batch", str(max_batch)]
        if lib:
            cmd += ["--lib", lib]
        e = dict(os.environ)
        e.update(env or {})
        self.proc = subprocess.Popen(cmd, env=e, stderr=subprocess.PIPE, text=True)

    def wait_ready(self, timeout_s: float = 60.0) -> None:
        deadline = time.time() + timeout_s
        while time.time() < deadline:
            if self.proc.poll() is not None:
                raise SidecarError(f"pgemb_sidecar exited with {self.proc.returncode}: {self.proc.stderr.read()[-2000:]}")
            if client().pgemb_client_connect(self.shm_name.encode(), 50) == 0:
                return
        self.stop()
        raise SidecarError("pgemb_sidecar did not start serving")

    def stop(self, timeout_s: float = 30.0) -> int:
        if self.proc.poll() is None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout_s)
            except subprocess.TimeoutExpired:
                self.proc.kill()
                self.proc.wait()
        return self.proc.returncode
