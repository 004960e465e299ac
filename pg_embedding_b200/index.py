"""Host-side mirror of the reference's interface for the hot path, above the C ABI.

Names follow the reference: the three SQL distance functions (embedding--0.3.6.sql:20-27,
embedding.c:1040-1062), the index options dims / m / efconstruction / efsearch (embedding.c:125-149),
insert = hnsw_add_point (embedding.c:606-701), scan = hnsw_gettuple with its efSearch doubling
(embedding.c:285-370).  Everything computes on the GPU through libpgemb_b200.so; importing this module
without the built extension raises (no CPU fallback).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import HnswMetadata, PgembHostIndex, check

DIST_L2, DIST_COSINE, DIST_MANHATTAN = 0, 1, 2
METRICS = {"l2": DIST_L2, "cosine": DIST_COSINE, "manhattan": DIST_MANHATTAN,
           # opclass names (embedding--0.3.6.sql:57-70)
           "ann_l2_ops": DIST_L2, "ann_cos_ops": DIST_COSINE, "ann_manhattan_ops": DIST_MANHATTAN}

DEFAULT_M, DEFAULT_EF_CONSTRUCT, DEFAULT_EF_SEARCH = 100, 16, 64  # embedding.c:111-113
DELETED_FLAG_BIT = 48  # HnswLabel.pg.flags & DELETED_FLAG (embedding.c:44, :50-56)
NO_LABEL = np.iinfo(np.uint64).max


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a, ct):
    return a.ctypes.data_as(C.POINTER(ct)) if a is not None else None


def _metric(m) -> int:
    return METRICS[m] if isinstance(m, str) else int(m)


def device_count() -> int:
    return int(_lib.load().pgemb_device_count())


# ---- SQL-callable distance functions (embedding.c:1022-1062) -------------------------------------
def _calc_distance(metric: int, a, b) -> np.float32:
    a, b = _f32(a).ravel(), _f32(b).ravel()
    if a.shape[0] != b.shape[0]:
        # embedding.c:1031-1035
        raise ValueError(f"different array dimensions {a.shape[0]} and {b.shape[0]}")
    lib = _lib.load()
    out = np.empty(1, dtype=np.float32)
    check(lib.pgemb_dist_batch(metric, a.shape[0], 1, _p(a, C.c_float), 0, _p(b, C.c_float), _p(out, C.c_float)))
    return out[0]


def l2_distance(a, b) -> np.float32:          # operator <->
    return _calc_distance(DIST_L2, a, b)


def cosine_distance(a, b) -> np.float32:      # operator <=>
    return _calc_distance(DIST_COSINE, a, b)


def manhattan_distance(a, b) -> np.float32:   # operator <~>
    return _calc_distance(DIST_MANHATTAN, a, b)


def dist_batch(metric, a, b) -> np.ndarray:
    """a: [dim] (broadcast) or [n, dim]; b: [n, dim] -> float32[n] (one hnsw_dist_func each, on the GPU)."""
    a, b = _f32(a), _f32(b)
    n, dim = b.shape
    if a.shape[-1] != dim:
        raise ValueError(f"different array dimensions {a.shape[-1]} and {dim}")
    out = np.empty(n, dtype=np.float32)
    check(_lib.load().pgemb_dist_batch(_metric(metric), dim, n, _p(a, C.c_float), int(a.ndim == 1),
                                       _p(b, C.c_float), _p(out, C.c_float)))
    return out


class HnswIndex:
    """`CREATE INDEX ... USING hnsw(col) WITH (dims=, m=, efconstruction=, efsearch=)` on a GPU."""

    def __init__(self, dims: int, m: int = DEFAULT_M, efconstruction: int = DEFAULT_EF_CONSTRUCT,
                 efsearch: int = DEFAULT_EF_SEARCH, metric="l2", capacity: int = 1 << 16, device: int = 0):
        self.lib = _lib.load()
        self.host = PgembHostIndex()
        check(self.lib.pgemb_meta_init(C.byref(self.host.meta), int(dims), int(m), int(efconstruction),
                                       int(efsearch), _metric(metric)))
        dev = C.c_void_p()
        check(self.lib.pgemb_index_create(C.byref(self.host.meta), int(capacity), int(device), C.byref(dev)))
        self.device = int(device)
        self.host.dev = dev.value
        self.dev = dev
        self.dims, self.m, self.maxm = int(dims), int(m), 2 * int(m)
        self.metric = _metric(metric)

    # -- lifecycle ---------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "dev", None) is not None and self.dev.value:
            self.lib.pgemb_index_destroy(self.dev)
            self.dev = C.c_void_p()
            self.host.dev = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return int(self.lib.pgemb_index_size(self.dev))

    @property
    def meta(self) -> HnswMetadata:
        return self.host.meta

    @property
    def efsearch(self) -> int:
        return int(self.host.meta.efSearch)

    @efsearch.setter
    def efsearch(self, v: int):
        self.host.meta.efSearch = int(v)

    @property
    def efconstruction(self) -> int:
        return int(self.host.meta.efConstruction)

    # -- storing nodes -----------------------------------------------------------------------------
    def _check_dims(self, v):
        if v.shape[-1] != self.dims:
            # embedding.c:177-181 / :311-315
            raise ValueError(f"Wrong number of dimensions: {v.shape[-1]} instead of {self.dims} expected")

    def append(self, vecs, labels=None, links=None) -> None:
        """Store nodes without binding them (zeroed link lists unless `links` is given)."""
        v = _f32(vecs).reshape(-1, np.shape(vecs)[-1])
        self._check_dims(v)
        lab = None if labels is None else np.ascontiguousarray(labels, dtype=np.uint64)
        lk = None
        if links is not None:
            lk = np.ascontiguousarray(links, dtype=np.uint32)
            assert lk.shape == (v.shape[0], self.maxm + 1)
        check(self.lib.pgemb_index_append(self.dev, v.shape[0], _p(v, C.c_float), _p(lab, C.c_uint64), _p(lk, C.c_uint32)))

    def insert(self, vec, label=None) -> None:
        """hnsw_add_point (embedding.c:606-701): store the record, then hnsw_bind_point through the
        reference-shaped entry point."""
        v = _f32(vec).ravel()
        self._check_dims(v)
        cur = len(self)
        self.append(v[None, :], None if label is None else [label])
        if not self.lib.hnsw_bind_point(C.byref(self.host.meta), _p(v, C.c_float), cur):
            raise RuntimeError("HNSW index insert failed: " + self.lib.pgemb_last_error().decode())  # embedding.c:187

    def insert_many(self, vecs, labels=None) -> None:
        """n sequential inserts with the exact reference semantics, bound on the device back to back."""
        v = _f32(vecs)
        self._check_dims(v)
        lab = None if labels is None else np.ascontiguousarray(labels, dtype=np.uint64)
        check(self.lib.pgemb_insert_batch(self.dev, v.shape[0], _p(v, C.c_float), _p(lab, C.c_uint64)))

    def build(self, vecs, labels=None, batch_max: int = 4096) -> float:
        """Bulk build (ambuild): append then pgemb_build_bulk. Returns device seconds of the bind phase."""
        first = len(self)
        self.append(vecs, labels)
        return self.build_appended(first, len(self) - first, batch_max)

    def build_appended(self, first: int, n: int, batch_max: int = 4096) -> float:
        secs = C.c_double(0)
        check(self.lib.pgemb_build_bulk(self.dev, int(first), int(n), int(batch_max), C.byref(secs)))
        return secs.value

    def build_exact(self, first: int, n: int, batch_max: int = 256):
        """Exact parallel build of already appended nodes: bit-identical to sequential inserts.
        Returns (device seconds, dict(batches, searches, inserts))."""
        secs = C.c_double(0)
        st = (C.c_uint64 * 3)()
        check(self.lib.pgemb_build_exact(self.dev, int(first), int(n), int(batch_max), C.byref(secs), st))
        return secs.value, {"batches": int(st[0]), "searches": int(st[1]), "inserts": int(st[2])}

    def load_records(self, records: np.ndarray) -> None:
        """Ingest nodes in the reference's on-page record layout (embedding.c:224-228)."""
        r = np.ascontiguousarray(records, dtype=np.uint8)
        check(self.lib.pgemb_index_append_records(self.dev, r.shape[0], r.ctypes.data_as(C.c_void_p), r.shape[1]))

    def export_records(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = len(self) - first if n is None else n
        rs = int(self.host.meta.size_data_per_element)
        out = np.zeros((n, rs), dtype=np.uint8)
        if n:
            check(self.lib.pgemb_index_export_records(self.dev, first, n, out.ctypes.data_as(C.c_void_p), rs))
        return out

    def links(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = len(self) - first if n is None else n
        out = np.zeros((n, self.maxm + 1), dtype=np.uint32)
        if n:
            check(self.lib.pgemb_index_get_links(self.dev, first, n, _p(out, C.c_uint32)))
        return out

    def set_links(self, links, first: int = 0) -> None:
        lk = np.ascontiguousarray(links, dtype=np.uint32)
        check(self.lib.pgemb_index_set_links(self.dev, first, lk.shape[0], _p(lk, C.c_uint32)))

    def labels(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = len(self) - first if n is None else n
        out = np.zeros(n, dtype=np.uint64)
        if n:
            check(self.lib.pgemb_index_get_labels(self.dev, first, n, _p(out, C.c_uint64)))
        return out

    def mark_deleted(self, ids, deleted: bool = True) -> None:
        """What ambulkdelete does to index entries (embedding.c:912-922)."""
        lab = self.labels()
        ids = np.asarray(ids, dtype=np.int64)
        bit = np.uint64(1) << np.uint64(DELETED_FLAG_BIT)
        if deleted:
            lab[ids] |= bit
        else:
            lab[ids] &= ~bit
        check(self.lib.pgemb_index_set_labels(self.dev, 0, lab.shape[0], _p(lab, C.c_uint64)))

    def truncate(self) -> None:
        check(self.lib.pgemb_index_truncate(self.dev))

    def reserve(self, capacity: int) -> None:
        """Grow the device index (a relation grows page by page); node ids and contents are preserved."""
        check(self.lib.pgemb_index_reserve(self.dev, int(capacity)))

    # -- searching ---------------------------------------------------------------------------------
    def search(self, q, efsearch: int | None = None) -> np.ndarray:
        """One hnsw_search call through the reference-shaped entry point (embedding.c:317)."""
        qv = _f32(q).ravel()
        self._check_dims(qv)
        if efsearch is not None:
            self.host.meta.efSearch = int(efsearch)
        n = C.c_size_t(0)
        res = C.POINTER(C.c_uint64)()
        if not self.lib.hnsw_search(C.byref(self.host.meta), _p(qv, C.c_float), C.byref(n), C.byref(res)):
            raise RuntimeError("HNSW index search failed: " + self.lib.pgemb_last_error().decode())  # embedding.c:318
        out = np.ctypeslib.as_array(res, shape=(max(n.value, 1),))[: n.value].copy()
        _libc_free(res)
        return out

    def search_batch(self, queries, efsearch: int | None = None, want_dists=True, want_ids=True, want_stats=False):
        """nq independent hnsw_search calls in one launch. Returns dict(labels, n, dists, ids, stats, kernel_ms)."""
        q = _f32(queries)
        self._check_dims(q)
        ef = self.efsearch if efsearch is None else int(efsearch)
        nq = q.shape[0]
        labels = np.empty((nq, ef), dtype=np.uint64)
        dists = np.empty((nq, ef), dtype=np.float32) if want_dists else None
        ids = np.empty((nq, ef), dtype=np.uint32) if want_ids else None
        stats = np.empty((nq, 4), dtype=np.uint32) if want_stats else None
        n = np.zeros(nq, dtype=np.int32)
        check(self.lib.pgemb_search_batch(self.dev, nq, _p(q, C.c_float), ef, _p(labels, C.c_uint64), _p(dists, C.c_float),
                                          _p(ids, C.c_uint32), _p(n, C.c_int32), _p(stats, C.c_uint32)))
        return {"labels": labels, "n": n, "dists": dists, "ids": ids, "stats": stats,
                "kernel_ms": float(self.lib.pgemb_last_kernel_ms(self.dev))}

    def scan(self, q, limit: int | None = None, efsearch: int | None = None, batch: int = 1):
        """hnsw_beginscan / hnsw_gettuple / hnsw_endscan (embedding.c:249-387) through the C ABI (pgemb_index_scan_*): yields
        heap TIDs (label without flags) until the scan is exhausted or `limit` tuples were returned.  batch > 1 fetches that many
        tuples per call (pgemb_index_scan_next_batch) -- same sequence."""
        qv = _f32(q).ravel()
        self._check_dims(qv)
        sc = C.c_void_p()
        check(self.lib.pgemb_index_scan_begin(self.dev, _p(qv, C.c_float), int(self.efsearch if efsearch is None else efsearch), C.byref(sc)))
        self.last_scan = {}
        try:
            returned = 0
            if batch <= 1:
                t = C.c_uint64(0)
                while limit is None or returned < limit:
                    r = self.lib.pgemb_index_scan_next(sc, C.byref(t))
                    if r < 0:
                        raise RuntimeError("HNSW index search failed: " + self.lib.pgemb_last_error().decode())  # embedding.c:318, :336
                    if r == 0:
                        return
                    returned += 1
                    yield int(t.value)
            else:
                buf = np.empty(batch, dtype=np.uint64)
                got = C.c_size_t(0)
                while limit is None or returned < limit:
                    want = batch if limit is None else min(batch, limit - returned)
                    check(self.lib.pgemb_index_scan_next_batch(sc, want, _p(buf, C.c_uint64), C.byref(got)))
                    for i in range(got.value):
                        returned += 1
                        yield int(buf[i])
                    if got.value < want:
                        return
        finally:
            self.last_scan = {"ef": int(self.lib.pgemb_index_scan_ef(sc)), "searches": int(self.lib.pgemb_index_scan_searches(sc))}
            self.lib.pgemb_index_scan_end(sc)

    def scan_topk(self, queries, k: int, metric=None):
        """Exact brute-force k-NN (the seq-scan answer, knn.out:63-91), batched. Returns dict(labels, dists, n).
        `metric` (name or DIST_*): the query's operator, any of the three; None = the index's own."""
        q = _f32(queries)
        self._check_dims(q)
        nq = q.shape[0]
        labels = np.empty((nq, k), dtype=np.uint64)
        dists = np.empty((nq, k), dtype=np.float32)
        n = np.zeros(nq, dtype=np.int32)
        out = (_p(q, C.c_float), int(k), _p(labels, C.c_uint64), _p(dists, C.c_float), _p(n, C.c_int32))
        if metric is None:
            check(self.lib.pgemb_scan_topk(self.dev, nq, *out))
        else:
            check(self.lib.pgemb_scan_topk_op(self.dev, _metric(metric), nq, *out))
        return {"labels": labels, "dists": dists, "n": n}

    def dist_gather(self, queries, ids) -> np.ndarray:
        q = _f32(queries)
        i = np.ascontiguousarray(ids, dtype=np.uint32)
        out = np.empty(i.shape, dtype=np.float32)
        check(self.lib.pgemb_dist_gather(self.dev, q.shape[0], _p(q, C.c_float), i.shape[1], _p(i, C.c_uint32), _p(out, C.c_float)))
        return out


_libc = C.CDLL(None)
_libc.free.argtypes = [C.c_void_p]


def _libc_free(ptr) -> None:
    _libc.free(C.cast(ptr, C.c_void_p))
