"""Throughput / latency of the reference-shaped hnsw_search (one query per call) when P backend PROCESSES call it at the
same time through pgemb_sidecar (the forked-backend deployment, DESIGN.md section 12) -- on an H100:

    python tools/bench_sidecar.py [--rows 1000000 --dims 768 --m 32 --metric cosine --backends 1,16,64,128 --seconds 5]

Prints one JSON line per backend count: aggregate queries/s, per-call latency percentiles, and how the sidecar batched
the calls (launches, mean and largest batch).  The graph is built once in the sidecar (bulk build); parity of the results
is checked by tests/test_sidecar.py, not here.

    python tools/bench_sidecar.py --op scan --k 10 [--backends 1,16,64,256]

measures the index-less plan instead (`ORDER BY val <op> q LIMIT k` without the index): every backend issues one
pgemb_client_scan_topk per call on the same table, no graph is built.  One JSON line per backend count (scans/s, latency
percentiles, pgemb_scan_topk calls, mean and largest batch), then two lines timing pgemb_scan_topk in this process on the
same table with nq = 1 and nq = 1024, for reference.  Every line names the GPU and its power limit.  Parity:
tests/test_sidecar_scan.py.

    python tools/bench_sidecar.py --op dist --dims 768 --metric cosine [--backends 1,16,64,256]

measures the SQL distance operators evaluated per row (one hnsw_dist_func per call on random pairs, no table): one JSON line
per backend count with distances/s, latency percentiles, pgemb_dist_batch calls, and mean and largest batch.

    python tools/bench_sidecar.py --op search+dist --k 10 [--backends 1,16,64,256]

models the projection query `SELECT id, val <=> q FROM t ORDER BY val <=> q LIMIT k` through the index: per call one
hnsw_search at --efs, then --k hnsw_dist_func calls between the query and the returned rows' vectors.  Reports queries/s.

    python tools/bench_sidecar.py --tree DIR ...

runs the sidecar, the client library and their Python binding of another source tree (for example a checkout of an earlier
commit, whose `pg_embedding_b200/build.py` builds its pgemb_sidecar and libpgemb_client.so), with this tree's
libpgemb_b200.so.  Client and server always come from the same tree: the protocol version is checked at connect.  A tree
without distance counters reports them as null; every line names the protocol version it ran.  Parity:
tests/test_sidecar_dist.py.
"""
import argparse
import ctypes as C
import json
import math
import os
import shutil
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
METRICS = {"l2": 0, "cosine": 1, "manhattan": 2}


def backend_main(a):
    """One backend: raw ctypes loop around hnsw_search (no numpy in the timed loop)."""
    sys.path.insert(0, os.path.abspath(a.tree))
    from pg_embedding_b200 import sidecar
    sidecar.connect(a.shm)
    lib = sidecar.client()
    if a.op == "dist":
        return dist_backend_loop(a, lib)
    idx = sidecar.RemoteIndex(1, a.dims, a.m, a.efc, a.efs, a.metric, capacity=1)
    rng = np.random.default_rng(1000 + a.backend_id)
    q = np.load(a.queries)
    q = np.ascontiguousarray(q[rng.permutation(q.shape[0])], dtype=np.float32)
    if a.op == "scan":
        return scan_backend_loop(a, idx, lib, q)
    rows = np.load(a.rows_file, mmap_mode="r") if a.op == "search+dist" else None   # the table, shared through the page cache
    metric = METRICS[a.metric]
    f32p = C.POINTER(C.c_float)
    free = C.CDLL(None).free
    free.argtypes = [C.c_void_p]
    n, res = C.c_size_t(), C.POINTER(C.c_uint64)()
    meta = C.byref(idx.h.meta)
    ptrs = [q[i].ctypes.data_as(C.POINTER(C.c_float)) for i in range(q.shape[0])]
    open(a.out + ".ready", "w").close()
    while not os.path.exists(a.go):
        time.sleep(0.001)
    lat = []
    t_end = time.perf_counter() + a.seconds
    i = 0
    while True:
        t0 = time.perf_counter()
        if t0 >= t_end:
            break
        qp = ptrs[i % len(ptrs)]
        if not lib.hnsw_search(meta, qp, C.byref(n), C.byref(res)):
            raise RuntimeError(lib.pgemb_client_last_error().decode())
        if rows is not None:
            # the projection: the executor evaluates `val <op> q` once per returned row (embedding.c:1022-1062)
            for j in range(min(a.k, n.value)):
                if math.isnan(lib.hnsw_dist_func(metric, rows[res[j]].ctypes.data_as(f32p), qp, a.dims)):
                    raise RuntimeError(lib.pgemb_client_last_error().decode())
        free(res)
        lat.append(time.perf_counter() - t0)
        i += 1
    np.save(a.out, np.array(lat, np.float64))


def scan_backend_loop(a, idx, lib, q):
    """One backend of --op scan: raw ctypes loop around pgemb_client_scan_topk (no numpy in the timed loop)."""
    f32p = C.POINTER(C.c_float)
    labels = (C.c_uint64 * a.k)()
    dists = (C.c_float * a.k)()
    n = C.c_size_t()
    h = C.byref(idx.h)
    ptrs = [q[i].ctypes.data_as(f32p) for i in range(q.shape[0])]
    open(a.out + ".ready", "w").close()
    while not os.path.exists(a.go):
        time.sleep(0.001)
    lat = []
    t_end = time.perf_counter() + a.seconds
    i = 0
    while True:
        t0 = time.perf_counter()
        if t0 >= t_end:
            break
        if lib.pgemb_client_scan_topk(h, ptrs[i % len(ptrs)], a.k, labels, dists, C.byref(n)) != 0:
            raise RuntimeError(lib.pgemb_client_last_error().decode())
        lat.append(time.perf_counter() - t0)
        i += 1
    np.save(a.out, np.array(lat, np.float64))


def dist_backend_loop(a, lib):
    """One backend of --op dist: raw ctypes loop around hnsw_dist_func on random pairs (no numpy in the timed loop)."""
    rng = np.random.default_rng(2000 + a.backend_id)
    pairs = rng.standard_normal((256, 2, a.dims)).astype(np.float32) + (1.0 if a.metric == "cosine" else 0.0)
    f32p = C.POINTER(C.c_float)
    ptrs = [(p[0].ctypes.data_as(f32p), p[1].ctypes.data_as(f32p)) for p in pairs]
    metric = METRICS[a.metric]
    open(a.out + ".ready", "w").close()
    while not os.path.exists(a.go):
        time.sleep(0.001)
    lat = []
    t_end = time.perf_counter() + a.seconds
    i = 0
    while True:
        t0 = time.perf_counter()
        if t0 >= t_end:
            break
        pa, pb = ptrs[i % len(ptrs)]
        if math.isnan(lib.hnsw_dist_func(metric, pa, pb, a.dims)):
            raise RuntimeError(lib.pgemb_client_last_error().decode())
        lat.append(time.perf_counter() - t0)
        i += 1
    np.save(a.out, np.array(lat, np.float64))


def gpu_info() -> dict:
    """The card's name and power limit (read-only nvidia-smi query): part of every figure this tool prints."""
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [f.strip() for f in out.split(",")]
        return {"gpu": name, "power_limit_w": float(plim)}
    except Exception:
        return {"gpu": None, "power_limit_w": None}


def time_in_process_scan(a, X, Q, info):
    """pgemb_scan_topk in this process on the sidecar's table (same rows, same metric): nq = 1 and nq = 1024."""
    import pg_embedding_b200 as pg
    idx = pg.HnswIndex(a.dims, a.m, a.efc, a.efs, a.metric, capacity=a.rows)
    step = 1 << 17
    for lo in range(0, a.rows, step):
        hi = min(a.rows, lo + step)
        idx.append(np.ascontiguousarray(X[lo:hi]), np.arange(lo, hi, dtype=np.uint64))
    for nq, reps in ((1, 200), (1024, 10)):
        q = np.ascontiguousarray(Q[:nq])
        idx.scan_topk(q, a.k)                                      # warm-up: module load, buffers of this shape
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            idx.scan_topk(q, a.k)                                  # host buffers: returns when the scan is done
            t.append(time.perf_counter() - t0)
        ms = float(np.median(t)) * 1e3
        print(json.dumps({"op": "scan", "in_process": True, "nq": nq, "k": a.k, "ms_per_call_median": round(ms, 3),
                          "scans_per_s": round(nq / (ms * 1e-3), 1), "calls": reps,
                          "workload": f"dims={a.dims} N={a.rows} {a.metric}, pgemb_scan_topk(nq={nq}) in one process, host buffers", **info}), flush=True)
    idx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dims", type=int, default=768)
    ap.add_argument("--m", type=int, default=32)
    ap.add_argument("--efc", type=int, default=200)
    ap.add_argument("--efs", type=int, default=64)
    ap.add_argument("--metric", default="cosine")
    ap.add_argument("--backends", default="1,16,64,128")
    ap.add_argument("--seconds", type=float, default=5.0)
    ap.add_argument("--linger-us", type=int, default=None, help="sidecar's --linger-us (default: the sidecar's own default)")
    ap.add_argument("--lib", default=None, help="C-ABI library the sidecar loads (default: the product library)")
    ap.add_argument("--op", choices=("search", "scan", "dist", "search+dist"), default="search",
                    help="search: hnsw_search per call; scan: pgemb_client_scan_topk per call; dist: hnsw_dist_func per call; "
                         "search+dist: hnsw_search then --k hnsw_dist_func per call")
    ap.add_argument("--k", type=int, default=10, help="LIMIT of --op scan, distances per query of --op search+dist")
    ap.add_argument("--tree", default=ROOT, help="source tree whose sidecar, client library and binding to run (default: this one)")
    ap.add_argument("--numpy-data", action="store_true", help="iid numpy data instead of bench.py's generator (no torch / CUDA in this process: emulated runs)")
    # internal: backend mode
    ap.add_argument("--backend-id", type=int, default=-1)
    ap.add_argument("--shm"), ap.add_argument("--queries"), ap.add_argument("--out"), ap.add_argument("--go"), ap.add_argument("--rows-file")
    a = ap.parse_args()
    if a.backend_id >= 0:
        return backend_main(a)

    from pg_embedding_b200 import build
    build.build()
    lib = a.lib
    if os.path.abspath(a.tree) != ROOT:
        # the other tree's sidecar and client over this tree's product library (whose kernels it then measures)
        lib = lib or build.OUT
        for m in [m for m in sys.modules if m == "pg_embedding_b200" or m.startswith("pg_embedding_b200.")]:
            del sys.modules[m]
        sys.path.insert(0, os.path.abspath(a.tree))
        from pg_embedding_b200 import build as tree_build
        tree_build.build_sidecar()
    from pg_embedding_b200 import sidecar
    assert os.path.dirname(os.path.abspath(sidecar.__file__)) == os.path.join(os.path.abspath(a.tree), "pg_embedding_b200")
    dist_stats = getattr(sidecar, "dist_stats", None)      # None: a tree without distance counters
    X = None
    if a.op == "dist":
        rng = np.random.default_rng(1234)
        X = np.zeros((0, a.dims), np.float32)               # no table: pairs are generated by the backends
        Q = rng.standard_normal((1, a.dims)).astype(np.float32)
    elif a.dims == 768 and not a.numpy_data:
        import bench  # the BASELINE data generator (clustered mixture, seeds 1234/5678)
        import torch
        X, Q = bench.make_data(torch, a.rows, 8192)
    if X is None:
        rng = np.random.default_rng(1234)
        X = rng.standard_normal((a.rows, a.dims)).astype(np.float32)
        Q = rng.standard_normal((8192, a.dims)).astype(np.float32)
    X = X.cpu().numpy() if hasattr(X, "cpu") else X
    Q = Q.cpu().numpy() if hasattr(Q, "cpu") else Q
    shm = f"/pgemb_bench_{os.getpid()}"
    srv = sidecar.SidecarProcess(shm, lib=lib, slots=512, bulk_mb=64, linger_us=a.linger_us)
    srv.wait_ready(120)
    tmp = f"/tmp/pgemb_bench_{os.getpid()}"
    os.makedirs(tmp, exist_ok=True)
    try:
        protocol = struct.unpack_from("<I", open("/dev/shm" + shm, "rb").read(8), 4)[0]
        idx = sidecar.RemoteIndex(1, a.dims, a.m, a.efc, a.efs, a.metric, capacity=max(X.shape[0], 1))
        rs = idx.record_bytes
        t0 = time.time()
        step = 16384  # 16384 x 3340 B = 55 MB per request: within the 64 MB bulk area
        for lo in range(0, X.shape[0], step):
            hi = min(X.shape[0], lo + step)
            rec = np.zeros((hi - lo, rs), np.uint8)
            rec[:, (2 * a.m + 1) * 4:(2 * a.m + 1) * 4 + a.dims * 4] = np.ascontiguousarray(X[lo:hi]).view(np.uint8)
            rec[:, rs - 8:] = np.arange(lo, hi, dtype=np.uint64).view(np.uint8).reshape(hi - lo, 8)
            idx.append_records(rec)
        t_ship = time.time() - t0
        if a.op in ("search", "search+dist"):
            t_build = idx.build(0, a.rows, batch_max=4096, exact=False)
            print(f"# shipped {a.rows} records in {t_ship:.1f}s, bulk build {t_build:.1f}s", file=sys.stderr)
        elif a.op == "scan":
            print(f"# shipped {a.rows} records in {t_ship:.1f}s (a scan needs no graph)", file=sys.stderr)
        info = gpu_info()
        qf, xf = os.path.join(tmp, "q.npy"), os.path.join(tmp, "x.npy")
        np.save(qf, Q)
        if a.op == "search+dist":
            np.save(xf, np.ascontiguousarray(X, dtype=np.float32))
        for P in [int(x) for x in a.backends.split(",")]:
            go = os.path.join(tmp, f"go{P}")
            s0 = sidecar.scan_stats() if a.op == "scan" else sidecar.stats()
            d0 = dist_stats() if dist_stats else None
            procs = []
            for b in range(P):
                out = os.path.join(tmp, f"lat_{P}_{b}.npy")
                cmd = [sys.executable, os.path.abspath(__file__), "--backend-id", str(b), "--shm", shm, "--queries", qf, "--out", out, "--go", go,
                       "--dims", str(a.dims), "--m", str(a.m), "--efc", str(a.efc), "--efs", str(a.efs), "--metric", a.metric, "--seconds", str(a.seconds),
                       "--op", a.op, "--k", str(a.k), "--tree", a.tree, "--rows-file", xf]
                procs.append((subprocess.Popen(cmd), out))
            while not all(os.path.exists(o + ".ready") or p.poll() is not None for p, o in procs):
                time.sleep(0.01)
            open(go, "w").close()
            for p, _ in procs:
                assert p.wait() == 0
            lat = np.concatenate([np.load(o) for _, o in procs])
            pct = {k: round(float(np.percentile(lat, v)) * 1e3, 3) for k, v in (("p50", 50), ("p90", 90), ("p99", 99))}
            if a.op == "scan":
                s1 = sidecar.scan_stats()
                nc, ns = s1["calls"] - s0["calls"], s1["scans"] - s0["scans"]
                print(json.dumps({"op": "scan", "backends": P, "k": a.k, "scans_per_s": round(lat.size / a.seconds, 1), "calls": int(lat.size),
                                  "latency_ms": pct, "scan_topk_calls": nc, "mean_batch": round(ns / max(nc, 1), 2), "max_batch_so_far": s1["max_batch"],
                                  "workload": f"dims={a.dims} N={a.rows} {a.metric} LIMIT {a.k}, one pgemb_client_scan_topk per call per backend process",
                                  **info}), flush=True)
                continue
            d1 = dist_stats() if dist_stats else None
            nd, ndc = (d1["dists"] - d0["dists"], d1["calls"] - d0["calls"]) if d1 else (None, None)
            dist_batching = {"dist_batch_calls": ndc, "mean_dist_batch": round(nd / max(ndc, 1), 2) if d1 else None,
                             "max_dist_batch_so_far": d1["max_batch"] if d1 else None, "protocol": protocol}
            if a.op == "dist":
                print(json.dumps({"op": "dist", "backends": P, "dists_per_s": round(lat.size / a.seconds, 1), "calls": int(lat.size),
                                  "latency_ms": pct, **dist_batching,
                                  "workload": f"dims={a.dims} {a.metric}, one hnsw_dist_func per call per backend process", **info}), flush=True)
                continue
            s1 = sidecar.stats()
            nb, ns = s1["batches"] - s0["batches"], s1["searches"] - s0["searches"]
            if a.op == "search+dist":
                print(json.dumps({"op": "search+dist", "backends": P, "k": a.k, "queries_per_s": round(lat.size / a.seconds, 1), "calls": int(lat.size),
                                  "latency_ms": pct, "launches": nb, "mean_batch": round(ns / max(nb, 1), 2), **dist_batching,
                                  "workload": f"dims={a.dims} N={a.rows} {a.metric} m={a.m} efS={a.efs}, per call one hnsw_search and "
                                              f"{a.k} hnsw_dist_func on the returned rows per backend process", **info}), flush=True)
                continue
            print(json.dumps({"backends": P, "queries_per_s": round(lat.size / a.seconds, 1), "calls": int(lat.size),
                              "latency_ms": pct,
                              "launches": nb, "mean_batch": round(ns / max(nb, 1), 2), "max_batch_so_far": s1["max_batch"],
                              "workload": f"dims={a.dims} N={a.rows} {a.metric} m={a.m} efS={a.efs}, one query per hnsw_search call per backend process"}))
        if a.op == "scan":
            time_in_process_scan(a, X, Q, info)
    finally:
        sidecar.client().pgemb_client_disconnect()
        srv.stop()
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
