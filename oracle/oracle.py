"""ctypes wrappers around the two CPU checkers.  TEST INFRASTRUCTURE ONLY.

* ``load("ref")``  -> oracle/_ref/libpgemb_ref.so  : the UNMODIFIED reference hnswalg.cpp + distfunc.c
  (compiled in place from /root/reference by oracle/Makefile) on our flat-memory host.
* ``load("port")`` -> oracle/_build/libpgemb_port.so: the C restatement oracle/hnsw_oracle.c on the
  same host.

Only tests/, ``__graft_entry__.smoke()`` and bench.py's cpu_baseline / ``--impl reference`` legs may
import this module; nothing under pg_embedding_b200/ does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.environ.get("PGEMB_REFERENCE_DIR", "/root/reference")

DIST_L2, DIST_COSINE, DIST_MANHATTAN = 0, 1, 2
METRICS = {"l2": DIST_L2, "cosine": DIST_COSINE, "manhattan": DIST_MANHATTAN}

_PATHS = {
    "ref": os.path.join(HERE, "_ref", "libpgemb_ref.so"),
    "port": os.path.join(HERE, "_build", "libpgemb_port.so"),
}
_LIBS: dict[str, C.CDLL] = {}


def build(which: str = "all", quiet: bool = True) -> None:
    """Compile the checkers (``make -C oracle``).  ``ref`` needs /root/reference and is skipped
    silently where that tree does not exist (the GPU box uses the prebuilt .so)."""
    targets = []
    if which in ("all", "port"):
        targets.append("port")
    if which in ("all", "ref") and os.path.isfile(os.path.join(REF_SRC, "hnswalg.cpp")):
        targets.append("ref")
    if not targets:
        return
    cmd = ["make", "-C", HERE, f"REF={REF_SRC}"] + targets
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"oracle build failed:\n{res.stdout}\n{res.stderr}")
    if not quiet:
        print(res.stdout)


def available(which: str) -> bool:
    return os.path.isfile(_PATHS[which])


def _f32p(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def load(which: str) -> C.CDLL:
    if which in _LIBS:
        return _LIBS[which]
    path = _PATHS[which]
    build(which)          # incremental (make): picks up edits of the checker sources; a no-op for `ref` where /root/reference is absent
    if not os.path.isfile(path):
        raise FileNotFoundError(f"{path} missing (build it here with `make -C oracle`)")
    lib = C.CDLL(path)
    vp, sz, f32p = C.c_void_p, C.c_size_t, C.POINTER(C.c_float)
    u64p, u32p, i32p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)
    lib.flat_create.restype = vp
    lib.flat_create.argtypes = [sz, sz, sz, sz, C.c_int, sz]
    lib.flat_destroy.argtypes = [vp]
    lib.flat_size.restype = sz
    lib.flat_size.argtypes = [vp]
    lib.flat_record_size.restype = sz
    lib.flat_record_size.argtypes = [vp]
    lib.flat_records.restype = vp
    lib.flat_records.argtypes = [vp]
    lib.flat_truncate.argtypes = [vp]
    lib.flat_add.restype = C.c_int
    lib.flat_add.argtypes = [vp, f32p, C.c_uint64]
    lib.flat_append_raw.restype = C.c_int
    lib.flat_append_raw.argtypes = [vp, sz, f32p, u64p, u32p]
    lib.flat_append_records.restype = C.c_int
    lib.flat_append_records.argtypes = [vp, sz, vp, sz]
    lib.flat_bind.restype = C.c_int
    lib.flat_bind.argtypes = [vp, C.c_uint32]
    lib.flat_get_links.argtypes = [vp, sz, sz, u32p]
    lib.flat_set_links.argtypes = [vp, sz, sz, u32p]
    lib.flat_get_coords.argtypes = [vp, sz, sz, f32p]
    lib.flat_get_labels.argtypes = [vp, sz, sz, u64p]
    lib.flat_set_label.argtypes = [vp, C.c_uint32, C.c_uint64]
    lib.flat_mark_deleted.argtypes = [vp, C.c_uint32, C.c_int]
    lib.flat_set_ef.argtypes = [vp, sz, sz]
    lib.flat_search.restype = C.c_long
    lib.flat_search.argtypes = [vp, f32p, sz, u64p]
    lib.flat_dist.restype = C.c_float
    lib.flat_dist.argtypes = [C.c_int, f32p, f32p, sz]
    lib.flat_dist_many.argtypes = [C.c_int, f32p, f32p, sz, sz, C.c_int, f32p]
    lib.flat_counters_reset.argtypes = []
    lib.flat_counters_get.argtypes = [u64p]
    lib.flat_search_many.restype = C.c_double
    lib.flat_search_many.argtypes = [vp, f32p, sz, sz, C.c_int, C.c_int, u64p, i32p, u64p]
    lib.flat_build.restype = C.c_double
    lib.flat_build.argtypes = [vp, sz, f32p, u64p]
    lib.flat_scan_begin.restype = vp
    lib.flat_scan_begin.argtypes = [vp, f32p, sz, sz]
    lib.flat_scan_next.restype = C.c_int
    lib.flat_scan_next.argtypes = [vp, u64p]
    lib.flat_scan_searches.restype = C.c_uint64
    lib.flat_scan_searches.argtypes = [vp]
    lib.flat_scan_ef.restype = sz
    lib.flat_scan_ef.argtypes = [vp]
    lib.flat_scan_end.argtypes = [vp]
    if which == "port":
        lib.oracle_cosine_norm.restype = C.c_float
        lib.oracle_cosine_norm.argtypes = [f32p, sz]
        lib.oracle_cosine_from_parts.restype = C.c_float
        lib.oracle_cosine_from_parts.argtypes = [f32p, f32p, sz]
        lib.oracle_search_ids.restype = C.c_long
        lib.oracle_search_ids.argtypes = [vp, f32p, sz, u32p, f32p]
        lib.oracle_bind_batch.restype = C.c_int
        lib.oracle_bind_batch.argtypes = [vp, C.c_uint32, sz]
    _LIBS[which] = lib
    return lib


def _metric(m) -> int:
    return METRICS[m] if isinstance(m, str) else int(m)


def dist(which: str, metric, a, b) -> np.float32:
    lib = load(which)
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    assert a.shape == b.shape and a.ndim == 1
    return np.float32(lib.flat_dist(_metric(metric), _f32p(a), _f32p(b), a.shape[0]))


def dist_many(which: str, metric, a, b) -> np.ndarray:
    """a: [dim] (broadcast) or [n, dim]; b: [n, dim] -> float32[n], one hnsw_dist_func call each."""
    lib = load(which)
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    n, dim = b.shape
    out = np.empty(n, dtype=np.float32)
    lib.flat_dist_many(_metric(metric), _f32p(a), _f32p(b), dim, n, int(a.ndim == 1), _f32p(out))
    return out


def bulk_schedule(first: int, n: int, batch_max: int) -> list:
    """pgemb_build_bulk's batches (capi.cu) over nodes [first, first+n) as (first node, size) pairs: a batch is at most 1/32 of
    the nodes before it (at least 1), at most batch_max (clamped to [1, 65536]) and never runs past the end; node 0 is skipped."""
    batch_max = min(max(int(batch_max), 1), 1 << 16)
    pos, end, out = int(first), int(first) + int(n), []
    while pos < end:
        if pos == 0:
            pos = 1             # node 0 has nothing to connect to
            continue
        b = min(max(pos // 32, 1), batch_max, end - pos)
        out.append((pos, b))
        pos += b
    return out


class FlatIndex:
    """The reference algorithm on a flat array of reference-layout records (see flat_host.c)."""

    def __init__(self, which: str, dims: int, m: int = 100, efconstruction: int = 16, efsearch: int = 64,
                 metric="l2", capacity: int = 1024):
        self.which = which
        self.lib = load(which)
        self.dims, self.m, self.maxm = int(dims), int(m), 2 * int(m)
        self.efc, self.efs = int(efconstruction), int(efsearch)
        self.metric = _metric(metric)
        self.capacity = int(capacity)
        self.h = self.lib.flat_create(self.dims, self.m, self.efc, self.efs, self.metric, self.capacity)
        if not self.h:
            raise MemoryError("flat_create failed")

    def close(self):
        if self.h:
            self.lib.flat_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return int(self.lib.flat_size(self.h))

    def add(self, vec, label: int | None = None) -> None:
        """hnsw_add_point: store record, bind (embedding.c:606-701)."""
        v = np.ascontiguousarray(vec, dtype=np.float32)
        assert v.shape == (self.dims,)
        lab = len(self) if label is None else int(label)
        rc = self.lib.flat_add(self.h, _f32p(v), lab)
        if rc != 0:
            raise RuntimeError(f"flat_add failed rc={rc}")

    def build(self, vecs, labels=None) -> float:
        v = np.ascontiguousarray(vecs, dtype=np.float32)
        assert v.ndim == 2 and v.shape[1] == self.dims
        lp = None
        if labels is not None:
            labels = np.ascontiguousarray(labels, dtype=np.uint64)
            lp = labels.ctypes.data_as(C.POINTER(C.c_uint64))
        t = self.lib.flat_build(self.h, v.shape[0], _f32p(v), lp)
        if t < 0:
            raise RuntimeError("flat_build failed")
        return t

    def load_graph(self, vecs, links, labels=None) -> None:
        """Append records with given link lists (no binding): search a graph built elsewhere."""
        v = np.ascontiguousarray(vecs, dtype=np.float32)
        l = np.ascontiguousarray(links, dtype=np.uint32)
        assert l.shape == (v.shape[0], self.maxm + 1)
        lp = None
        if labels is not None:
            labels = np.ascontiguousarray(labels, dtype=np.uint64)
            lp = labels.ctypes.data_as(C.POINTER(C.c_uint64))
        rc = self.lib.flat_append_raw(self.h, v.shape[0], _f32p(v), lp, l.ctypes.data_as(C.POINTER(C.c_uint32)))
        if rc != 0:
            raise RuntimeError("flat_append_raw failed (capacity?)")

    def load_records(self, records) -> None:
        """Append nodes given in the reference record layout [n, record_size] uint8."""
        r = np.ascontiguousarray(records, dtype=np.uint8)
        rc = self.lib.flat_append_records(self.h, r.shape[0], r.ctypes.data_as(C.c_void_p), r.shape[1])
        if rc != 0:
            raise RuntimeError("flat_append_records failed (capacity / stride?)")

    def append_unbound(self, vecs, labels=None) -> None:
        v = np.ascontiguousarray(vecs, dtype=np.float32)
        lp = None
        if labels is not None:
            labels = np.ascontiguousarray(labels, dtype=np.uint64)
            lp = labels.ctypes.data_as(C.POINTER(C.c_uint64))
        rc = self.lib.flat_append_raw(self.h, v.shape[0], _f32p(v), lp, None)
        if rc != 0:
            raise RuntimeError("flat_append_raw failed (capacity?)")

    def bind(self, idx: int) -> None:
        rc = self.lib.flat_bind(self.h, int(idx))
        if rc != 0:
            raise RuntimeError(f"bind failed rc={rc}")

    def build_bulk(self, first: int, n: int, batch_max: int = 4096) -> list:
        """(port only) pgemb_build_bulk's result on the stored, unbound nodes [first, first+n): its batch schedule (capi.cu) with
        every batch bound by oracle_bind_batch.  Returns the batch sizes in order."""
        if self.which != "port":
            raise ValueError("build_bulk is a model stated with the C restatement's primitives: port only")
        sizes = []
        for pos, b in bulk_schedule(first, n, batch_max):
            if self.lib.oracle_bind_batch(self.h, pos, b) != 0:
                raise RuntimeError(f"bind batch [{pos}, {pos + b}) failed")
            sizes.append(b)
        return sizes

    def links(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = len(self) - first if n is None else n
        out = np.zeros((n, self.maxm + 1), dtype=np.uint32)
        if n:
            self.lib.flat_get_links(self.h, first, n, out.ctypes.data_as(C.POINTER(C.c_uint32)))
        return out

    def set_links(self, links, first: int = 0) -> None:
        l = np.ascontiguousarray(links, dtype=np.uint32)
        self.lib.flat_set_links(self.h, first, l.shape[0], l.ctypes.data_as(C.POINTER(C.c_uint32)))

    def coords(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = len(self) - first if n is None else n
        out = np.zeros((n, self.dims), dtype=np.float32)
        if n:
            self.lib.flat_get_coords(self.h, first, n, _f32p(out))
        return out

    def labels(self, first: int = 0, n: int | None = None) -> np.ndarray:
        n = len(self) - first if n is None else n
        out = np.zeros(n, dtype=np.uint64)
        if n:
            self.lib.flat_get_labels(self.h, first, n, out.ctypes.data_as(C.POINTER(C.c_uint64)))
        return out

    def records(self) -> np.ndarray:
        """The raw AoS record bytes [n, record_size] (a copy)."""
        n, rs = len(self), int(self.lib.flat_record_size(self.h))
        buf = (C.c_char * (n * rs)).from_address(self.lib.flat_records(self.h))
        return np.frombuffer(buf, dtype=np.uint8).reshape(n, rs).copy()

    def mark_deleted(self, idx: int, deleted: bool = True) -> None:
        self.lib.flat_mark_deleted(self.h, int(idx), int(deleted))

    def truncate(self) -> None:
        self.lib.flat_truncate(self.h)

    def set_ef(self, efconstruction=None, efsearch=None) -> None:
        if efconstruction is not None:
            self.efc = int(efconstruction)
        if efsearch is not None:
            self.efs = int(efsearch)
        self.lib.flat_set_ef(self.h, self.efc, self.efs)

    def search(self, q, efsearch: int | None = None) -> np.ndarray:
        """One hnsw_search call: labels ascending by distance, deleted filtered."""
        ef = self.efs if efsearch is None else int(efsearch)
        qv = np.ascontiguousarray(q, dtype=np.float32)
        assert qv.shape == (self.dims,)
        out = np.empty(max(ef, 1), dtype=np.uint64)
        n = self.lib.flat_search(self.h, _f32p(qv), ef, out.ctypes.data_as(C.POINTER(C.c_uint64)))
        if n < 0:
            raise RuntimeError("hnsw_search failed")
        return out[:n].copy()

    def scan(self, q, efsearch: int | None = None, limit: int | None = None) -> dict:
        """hnsw_gettuple's iteration (embedding.c:285-370; oracle/scan_iter.c) until it returns false or `limit` tuples:
        dict(tids = the heap TIDs in the order handed out, searches = hnsw_search calls made, ef = final efSearch)."""
        ef = self.efs if efsearch is None else int(efsearch)
        qv = np.ascontiguousarray(q, dtype=np.float32)
        assert qv.shape == (self.dims,)
        sc = self.lib.flat_scan_begin(self.h, _f32p(qv), self.dims, ef)
        out, t = [], C.c_uint64(0)
        try:
            while limit is None or len(out) < limit:
                r = self.lib.flat_scan_next(sc, C.byref(t))
                if r < 0:
                    raise RuntimeError("HNSW index search failed")
                if r == 0:
                    break
                out.append(t.value)
            return {"tids": np.array(out, dtype=np.uint64), "searches": int(self.lib.flat_scan_searches(sc)), "ef": int(self.lib.flat_scan_ef(sc))}
        finally:
            self.lib.flat_scan_end(sc)

    def search_ids(self, q, efsearch: int | None = None):
        """(port only) internal ids + distances of searchBaseLayer's result, ascending (dist, id)."""
        assert self.which == "port"
        ef = self.efs if efsearch is None else int(efsearch)
        qv = np.ascontiguousarray(q, dtype=np.float32)
        ids = np.empty(max(ef, 1), dtype=np.uint32)
        ds = np.empty(max(ef, 1), dtype=np.float32)
        n = self.lib.oracle_search_ids(self.h, _f32p(qv), ef, ids.ctypes.data_as(C.POINTER(C.c_uint32)), _f32p(ds))
        return ids[:n].copy(), ds[:n].copy()

    def search_many(self, queries, efsearch: int | None = None, nthreads: int = 1, reps: int = 1,
                    want_labels: bool = True, want_counters: bool = False):
        """Timed multi-threaded search.  Returns dict(seconds, labels[nq,ef], n[nq], counters[nq,3])."""
        ef = self.efs if efsearch is None else int(efsearch)
        q = np.ascontiguousarray(queries, dtype=np.float32)
        nq = q.shape[0]
        labels = np.full((nq, ef), np.iinfo(np.uint64).max, dtype=np.uint64) if want_labels else None
        n_out = np.zeros(nq, dtype=np.int32)
        counters = np.zeros((nq, 3), dtype=np.uint64) if want_counters else None
        secs = self.lib.flat_search_many(
            self.h, _f32p(q), nq, ef, int(nthreads), int(reps),
            labels.ctypes.data_as(C.POINTER(C.c_uint64)) if labels is not None else None,
            n_out.ctypes.data_as(C.POINTER(C.c_int32)),
            counters.ctypes.data_as(C.POINTER(C.c_uint64)) if counters is not None else None)
        if secs < 0:
            raise RuntimeError("flat_search_many failed")
        return {"seconds": secs, "labels": labels, "n": n_out, "counters": counters}
