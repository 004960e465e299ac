"""The index-less scan through pgemb_sidecar: `SET enable_indexscan = off; SELECT ... ORDER BY val <op> q LIMIT k` in the
forked-backend deployment (DESIGN.md section 12, INTEGRATION.md section 7).

Each backend process calls pgemb_client_scan_topk with one query; the sidecar gathers the scans pending at the same time
per (relation, k) into one pgemb_scan_topk call.  What must hold: every result is the oracle's -- hnsw_dist_func's
distances (oracle.dist_many) sorted by (dist, label), deleted labels skipped, labels and distance BITS equal -- whatever
the interleaving; concurrent scans share calls; scans leave the search counters alone; a scan sees the writes that
completed before it; errors, cancellation and a dead sidecar behave as for hnsw_search.

CPU suite: the sidecar dlopen()s the host-emulated build of the C-ABI library (tests/emu).  `-m gpu`: the same through
the real libpgemb_b200.so on an H100, at a size where the default policy takes the tensor-core filter."""
import json
import os
import signal
import struct
import subprocess
import sys
import time

import numpy as np
import pytest

pytestmark = pytest.mark.timeout(900, method="thread")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
KNN = [c for c in json.load(open(os.path.join(HERE, "golden", "kat_regress.json")))["cases"] if c["name"] == "knn"][0]
DELETED = np.uint64(1 << 48)
EMU_ENV = {"PGEMB_EMU_SMS": "2", "PGEMB_EMU_TMA": "late"}
PGEMB_ERR_ARG, PGEMB_CLIENT_INTERRUPTED = 2, 100


def _start(lib, name, env=None, **kw):
    from pg_embedding_b200 import build, sidecar
    build.build_sidecar()
    srv = sidecar.SidecarProcess(name, lib=lib, env=env, **kw)
    srv.wait_ready(120)
    return srv


def _shm_name():
    return f"/pgemb_scan_{os.getpid()}_{int(time.time() * 1e3) % 100000}"


@pytest.fixture(scope="module")
def emulated_lib(tmp_path_factory):
    from emu_build import build_emulated
    return build_emulated(tmp_path_factory.mktemp("emu_sidecar_scan"))


def _serve(lib, env=None, **kw):
    """A sidecar (limits of the CPU suite unless overridden) with this process connected to it."""
    from pg_embedding_b200 import sidecar
    opts = dict(slots=16, max_dim=64, max_ef=64, bulk_mb=1, linger_us=20000)
    opts.update(kw)
    sidecar.client().pgemb_client_disconnect()
    name = _shm_name()
    srv = _start(lib, name, env=env, **opts)
    sidecar.connect(name)
    return name, srv


def _stop(srv):
    from pg_embedding_b200 import sidecar
    sidecar.client().pgemb_client_disconnect()
    assert srv.stop() == 0, srv.proc.stderr.read()[-2000:]


@pytest.fixture()
def served(emulated_lib):
    from pg_embedding_b200 import sidecar
    name, srv = _serve(emulated_lib, env=EMU_ENV)
    yield sidecar, name
    _stop(srv)


# ---- tables and the oracle -------------------------------------------------------------------------------------------
def _tid_label(blk, pos, flags=0):
    return (blk >> 16) | ((blk & 0xFFFF) << 16) | (pos << 32) | (flags << 48)     # ItemPointerData + flags (embedding.c:44-56)


def _table(rng, n, dims, metric):
    """n rows, TID-shaped labels in shuffled order, every 9th row deleted."""
    x = rng.standard_normal((n, dims)).astype(np.float32) + (1.0 if metric == "cosine" else 0.0)
    labels = np.array([_tid_label(3 + i // 7, 1 + i % 7) for i in rng.permutation(n)], np.uint64)
    alive = np.arange(n) % 9 != 0
    return x, labels, alive


def _records(idx, x, labels):
    """The reference's on-page records [count|links[maxM]|coords|label] (embedding.c:224-228), links left empty: a scan reads
    coordinates and labels only."""
    n, dims, m, rs = x.shape[0], idx.dims, int(idx.h.meta.M), idx.record_bytes
    rec = np.zeros((n, rs), np.uint8)
    rec[:, (2 * m + 1) * 4:(2 * m + 1) * 4 + dims * 4] = np.ascontiguousarray(x, np.float32).view(np.uint8)
    rec[:, rs - 8:] = np.ascontiguousarray(labels, np.uint64).view(np.uint8).reshape(n, 8)
    return rec


def _mirror(sc, rel_key, x, labels, alive, metric, m=3):
    idx = sc.RemoteIndex(rel_key, x.shape[1], m, 8, 16, metric, capacity=x.shape[0])
    idx.append_records(_records(idx, x, np.where(alive, labels, labels | DELETED)))
    return idx


def oracle_topk(oracle_mod, metric, x, labels, alive, q, k):
    """hnsw_dist_func per row (the oracle's restatement), live rows sorted by (dist, label): labels and fp32 bits."""
    d = np.asarray(oracle_mod.dist_many("port", metric, q, x), np.float32)
    b = d.view(np.uint32)
    key = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000))     # the float order of the bit pattern
    order = np.lexsort((labels, key))
    order = order[alive[order]][:k]
    return {"labels": labels[order].tolist(), "dists": d[order].view(np.uint32).tolist()}


def _row(r):
    return {"labels": r["labels"][: r["n"]].tolist(), "dists": r["dists"][: r["n"]].view(np.uint32).tolist()}


def _slots_free(name, timeout_s=2.0):
    """Every request slot FREE (within timeout_s: the sidecar frees an abandoned slot right after the call that served it)."""
    deadline = time.time() + timeout_s
    while True:
        raw = open("/dev/shm" + name, "rb").read()
        n_slots, stride, slots_off = struct.unpack_from("<I", raw, 8)[0], struct.unpack_from("<I", raw, 20)[0], struct.unpack_from("<Q", raw, 24)[0]
        if all(struct.unpack_from("<I", raw, slots_off + i * stride)[0] == 0 for i in range(n_slots)):
            return True
        if time.time() > deadline:
            return False
        time.sleep(0.01)


# ---- backend processes -----------------------------------------------------------------------------------------------
class Blocker:
    """Keeps the sidecar busy for a while: another backend process runs an exact build (a control request of seconds on the
    emulated library).  Requests submitted meanwhile queue up and are served together by the next pass, which makes the
    batching and cancellation tests independent of process start-up timing."""

    def __init__(self, sc, name, rel_key, n=120):
        rng = np.random.default_rng(rel_key)
        x = rng.standard_normal((n, 8)).astype(np.float32)
        idx = sc.RemoteIndex(rel_key, 8, 3, 10, 16, "l2", capacity=n)
        idx.append_records(_records(idx, x, np.arange(n, dtype=np.uint64)))
        code = ("import sys; sys.path.insert(0, sys.argv[1])\n"
                "from pg_embedding_b200 import sidecar\n"
                "sidecar.connect(sys.argv[2])\n"
                "sidecar.RemoteIndex(int(sys.argv[3]), 8, 3, 10, 16, 'l2', capacity=1).build(0, int(sys.argv[4]), batch_max=32, exact=True)\n")
        self.name = name
        self.proc = subprocess.Popen([sys.executable, "-c", code, ROOT, name, str(rel_key), str(n)], stderr=subprocess.PIPE, text=True)

    def wait_busy(self, timeout_s=60.0):
        """Until the sidecar works on the build (a slot in state BUSY with op PGEMB_OP_BUILD)."""
        deadline = time.time() + timeout_s
        while time.time() < deadline:
            raw = open("/dev/shm" + self.name, "rb").read()
            n_slots, stride, slots_off = struct.unpack_from("<I", raw, 8)[0], struct.unpack_from("<I", raw, 20)[0], struct.unpack_from("<Q", raw, 24)[0]
            if any(struct.unpack_from("<II", raw, slots_off + i * stride) == (3, 12) for i in range(n_slots)):
                return
            assert self.proc.poll() is None, self.proc.stderr.read()[-2000:]
            time.sleep(0.001)
        raise AssertionError("the blocking build never started")

    def join(self):
        _, err = self.proc.communicate(timeout=600)
        assert self.proc.returncode == 0, err[-2000:]


def _run_backends(shm, rel_key, cfg, jobs, tmp_path, blocker=None, during=None):
    """One backend process per job (op, k_or_ef, queries), all started together; with `blocker` (a function returning a
    Blocker), while the sidecar is busy.  `during()` runs in this process while the backends run."""
    procs = []
    for p, (op, k, q) in enumerate(jobs):
        qf, of = str(tmp_path / f"q{p}.npy"), str(tmp_path / f"out{p}.json")
        np.save(qf, q)
        cmd = [sys.executable, os.path.join(HERE, "sidecar_scan_backend.py"), shm, str(rel_key)] + [str(c) for c in cfg] + [op, str(k), qf, of]
        procs.append((subprocess.Popen(cmd, stderr=subprocess.PIPE, text=True), of))
    deadline = time.time() + 300
    while not all(os.path.exists(of + ".ready") or pr.poll() is not None for pr, of in procs) and time.time() < deadline:
        time.sleep(0.01)
    if blocker is not None:
        blocker = blocker()
        blocker.wait_busy()
    open(str(tmp_path / "go"), "w").close()
    if during is not None:
        during()
    got = []
    for pr, of in procs:
        _, err = pr.communicate(timeout=600)
        assert pr.returncode == 0, err[-2000:]
        got.append(json.load(open(of)))
    if blocker is not None:
        blocker.join()
    return got


# ---- bodies shared by the CPU suite and -m gpu ---------------------------------------------------------------------------
def check_knn_seqscan(sc, oracle_mod, rel_base=5000):
    """knn.out:63-91: the regress table's seq-scan order for <->, <=> and <~>, LIMIT 4, through pgemb_client_scan_topk."""
    rows = KNN["rows"]
    x = np.array([r["val"] for r in rows], np.float32)
    labels = np.array([_tid_label(*r["tid"]) for r in rows], np.uint64)
    alive = np.ones(len(rows), bool)
    q = np.array(KNN["query"], np.float32)
    for mi, (metric, want) in enumerate(KNN["expected"].items()):
        idx = _mirror(sc, rel_base + mi, x, labels, alive, metric)
        got = idx.scan_topk(q, 4)
        by_label = {int(l): r["val"] for l, r in zip(labels, rows)}
        assert [by_label[int(l)] for l in got["labels"][: got["n"]]] == want, metric
        assert _row(got) == oracle_topk(oracle_mod, metric, x, labels, alive, q, 4), metric
        idx.drop()


def check_concurrent_scans(sc, name, oracle_mod, metric, n, dims, ks, per, tmp_path, blocker=False, rel_key=42):
    """len(ks) backend processes, `per` scans each, backend p with LIMIT ks[p]: every result is the oracle's, the
    sidecar served them in fewer pgemb_scan_topk calls than scans, and the search counters did not move.  `blocker`: the
    backends start while the sidecar is busy (Blocker), so their first scans are certain to meet in one pass."""
    rng = np.random.default_rng([n, dims, ("l2", "cosine", "manhattan").index(metric)])
    x, labels, alive = _table(rng, n, dims, metric)
    idx = _mirror(sc, rel_key, x, labels, alive, metric)
    P = len(ks)
    q = rng.standard_normal((P * per, dims)).astype(np.float32) + (1.0 if metric == "cosine" else 0.0)
    s0, c0 = sc.stats(), sc.scan_stats()
    jobs = [("scan", ks[p], q[p * per:(p + 1) * per]) for p in range(P)]
    got = _run_backends(name, rel_key, (dims, 3, 8, 16, metric), jobs, tmp_path, blocker=(lambda: Blocker(sc, name, 900)) if blocker else None)
    for p in range(P):
        for i in range(per):
            assert got[p][i] == oracle_topk(oracle_mod, metric, x, labels, alive, q[p * per + i], ks[p]), (metric, p, i)
    c1 = sc.scan_stats()
    assert c1["scans"] - c0["scans"] == P * per, c1
    assert c1["calls"] - c0["calls"] < P * per and c1["max_batch"] >= 2, (c0, c1)     # concurrent scans shared calls
    s1 = sc.stats()
    assert (s1["batches"], s1["searches"], s1["max_batch"]) == (s0["batches"], s0["searches"], s0["max_batch"]), (s0, s1)
    idx.drop()
    return c1


# ---- CPU suite (emulated library) --------------------------------------------------------------------------------------
def test_knn_regress_seqscan_through_the_sidecar(served, oracle_mod):
    sc, _ = served
    check_knn_seqscan(sc, oracle_mod)


@pytest.mark.parametrize("metric", ["l2", "cosine", "manhattan"])
def test_concurrent_scans_get_the_oracle_results(served, oracle_mod, metric, tmp_path):
    """4 backends x 6 scans, LIMIT 1 / 5 / 10 / 5: two backends share the (relation, k = 5) group."""
    sc, name = served
    c = check_concurrent_scans(sc, name, oracle_mod, metric, 300, 16, (1, 5, 10, 5), 6, tmp_path,
                               blocker=True)
    assert c["scans"] == 24


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_concurrent_scans_on_the_tensor_core_path(emulated_lib, oracle_mod, metric, tmp_path):
    """The same with the sidecar's scans forced through the tensor-core filter (PGEMB_SCAN_TC=2)."""
    from pg_embedding_b200 import sidecar
    name, srv = _serve(emulated_lib, env=dict(EMU_ENV, PGEMB_SCAN_TC="2"))
    try:
        check_concurrent_scans(sidecar, name, oracle_mod, metric, 300, 16, (1, 5, 10, 5), 6, tmp_path,
                               blocker=True)
    finally:
        _stop(srv)


def test_scan_groups_larger_than_max_batch_are_split(emulated_lib, oracle_mod, tmp_path):
    """--max-batch 2 and five concurrent scans of one (relation, k): served in calls of at most two, answers unchanged."""
    from pg_embedding_b200 import sidecar
    name, srv = _serve(emulated_lib, env=EMU_ENV, max_batch=2)
    try:
        rng = np.random.default_rng(15)
        n, dims, k, P, per = 200, 10, 7, 5, 3
        x, labels, alive = _table(rng, n, dims, "l2")
        idx = _mirror(sidecar, 21, x, labels, alive, "l2")
        q = rng.standard_normal((P * per, dims)).astype(np.float32)
        jobs = [("scan", k, q[p * per:(p + 1) * per]) for p in range(P)]
        got = _run_backends(name, 21, (dims, 3, 8, 16, "l2"), jobs, tmp_path, blocker=lambda: Blocker(sidecar, name, 901))
        for p in range(P):
            for i in range(per):
                assert got[p][i] == oracle_topk(oracle_mod, "l2", x, labels, alive, q[p * per + i], k), (p, i)
        st = sidecar.scan_stats()
        assert st["scans"] == P * per and st["max_batch"] == 2 and st["calls"] >= (P * per + 1) // 2, st
        idx.drop()
    finally:
        _stop(srv)


def test_mixed_search_and_scan_traffic_and_read_your_writes(served, oracle_mod, tmp_path):
    """Searching and scanning backends at once on one relation, while this process inserts rows into another and scans
    it right after each insert returned: every answer is the oracle's, and each scan sees the row just inserted."""
    sc, name = served
    rng = np.random.default_rng(23)
    n, dims, m, efc, ef, k = 300, 12, 4, 16, 12, 6
    x = rng.standard_normal((n, dims)).astype(np.float32)
    labels = np.array([_tid_label(3 + i // 7, 1 + i % 7) for i in rng.permutation(n)], np.uint64)
    alive = np.arange(n) % 9 != 0
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, "l2", capacity=n)
    orc.build(x, labels)
    for i in np.flatnonzero(~alive):
        orc.mark_deleted(int(i))
    idx = sc.RemoteIndex(51, dims, m, efc, 64, "l2", capacity=n)
    idx.append_records(orc.records())                               # the graph, for the searchers
    q = rng.standard_normal((4 * 5, dims)).astype(np.float32)
    jobs = [("search", ef, q[0:5]), ("scan", k, q[5:10]), ("search", ef, q[10:15]), ("scan", k, q[15:20])]

    w_dims, w_n = 6, 10
    wx = rng.standard_normal((w_n, w_dims)).astype(np.float32)
    wl = np.arange(700, 700 + w_n, dtype=np.uint64)
    w = sc.RemoteIndex(52, w_dims, 3, 8, 16, "l2", capacity=2)

    def writer():
        for i in range(w_n):
            w.append_records(_records(w, wx[i:i + 1], wl[i:i + 1]))  # the relation's new page record (embedding.c:619-621) ...
            w.bind_point(i)                                          # ... and hnsw_bind_point (:695) have returned
            got = w.scan_topk(wx[i], 4)
            assert _row(got) == oracle_topk(oracle_mod, "l2", wx[:i + 1], wl[:i + 1], np.ones(i + 1, bool), wx[i], 4), i
            assert int(wl[i]) in got["labels"][: got["n"]].tolist()

    got = _run_backends(name, 51, (dims, m, efc, 64, "l2"), jobs, tmp_path, during=writer)
    want_search = orc.search_many(q, ef)
    for p, (op, kk, _) in enumerate(jobs):
        for i in range(5):
            j = p * 5 + i
            if op == "search":
                assert got[p][i] == want_search["labels"][j, : want_search["n"][j]].tolist(), (p, i)
            else:
                assert got[p][i] == oracle_topk(oracle_mod, "l2", x, labels, alive, q[j], kk), (p, i)
    assert sc.stats()["searches"] == 10 and sc.scan_stats()["scans"] == 10 + w_n
    idx.drop()
    w.drop()


def test_scan_errors_leave_the_sidecar_serving(served, oracle_mod):
    """k = 0 and k beyond the sidecar's --max-ef are refused before a slot is claimed, an unattached relation by the
    sidecar; each with PGEMB_ERR_ARG and a message, and the next call succeeds with no slot leaked."""
    sc, name = served
    rng = np.random.default_rng(6)
    x, labels, alive = _table(rng, 50, 8, "l2")
    idx = _mirror(sc, 7, x, labels, alive, "l2")
    with pytest.raises(sc.SidecarError, match=f"pgemb status {PGEMB_ERR_ARG}: .*k = 0 outside 1 .. 64"):
        idx.scan_topk(x[0], 0)
    with pytest.raises(sc.SidecarError, match=f"pgemb status {PGEMB_ERR_ARG}: .*k = 65 outside 1 .. 64"):
        idx.scan_topk(x[0], 65)
    ghost = sc.RemoteIndex.__new__(sc.RemoteIndex)
    ghost.h = sc.PgembClientIndex()
    ghost.h.meta, ghost.h.rel_key, ghost.dims = idx.h.meta, 999, 8
    with pytest.raises(sc.SidecarError, match=f"pgemb status {PGEMB_ERR_ARG}: no device index attached"):
        ghost.scan_topk(x[0], 4)
    assert _row(idx.scan_topk(x[1], 64)) == oracle_topk(oracle_mod, "l2", x, labels, alive, x[1], 64)     # fewer live rows than k
    assert _slots_free(name)
    st = sc.scan_stats()
    assert st["scans"] == 1 and st["calls"] == 1, st        # nothing was scanned for the refused requests


def test_cancelled_scan_returns_and_the_sidecar_frees_its_slot(served, oracle_mod):
    """Query cancel while the scan waits behind another backend's long request: the call gives up with
    PGEMB_CLIENT_INTERRUPTED, the sidecar later runs the abandoned scan, drops its result and frees the slot."""
    import ctypes as C
    sc, name = served
    rng = np.random.default_rng(12)
    x, labels, alive = _table(rng, 80, 8, "l2")
    idx = _mirror(sc, 31, x, labels, alive, "l2")
    blocker = Blocker(sc, name, 902)
    blocker.wait_busy()
    pending = C.c_int(1)
    cb = C.CFUNCTYPE(C.c_int)(lambda: pending.value)
    sc.client().pgemb_client_set_interrupt_check(C.cast(cb, C.c_void_p))
    try:
        t0 = time.time()
        with pytest.raises(sc.SidecarError, match=f"pgemb status {PGEMB_CLIENT_INTERRUPTED}: interrupted"):
            idx.scan_topk(x[0], 5)
        assert time.time() - t0 < 2.0
        pending.value = 0
    finally:
        sc.client().pgemb_client_set_interrupt_check(None)
    blocker.join()
    assert _row(idx.scan_topk(x[2], 5)) == oracle_topk(oracle_mod, "l2", x, labels, alive, x[2], 5)
    assert sc.scan_stats()["scans"] == 2                   # the abandoned scan was run, too
    assert _slots_free(name), "a slot was leaked"


def test_scan_does_not_hang_when_the_sidecar_dies(emulated_lib, oracle_mod):
    from pg_embedding_b200 import sidecar
    name, srv = _serve(emulated_lib, env=EMU_ENV, slots=4, max_dim=16, max_ef=16)
    rng = np.random.default_rng(3)
    x, labels, alive = _table(rng, 50, 8, "l2")
    idx = _mirror(sidecar, 5, x, labels, alive, "l2")
    assert _row(idx.scan_topk(x[0], 3)) == oracle_topk(oracle_mod, "l2", x, labels, alive, x[0], 3)
    srv.proc.send_signal(signal.SIGKILL)
    srv.proc.wait()
    t0 = time.time()
    with pytest.raises(sidecar.SidecarError, match="no sidecar is serving"):
        idx.scan_topk(x[0], 3)
    assert time.time() - t0 < 5.0
    sidecar.client().pgemb_client_disconnect()
    if os.path.exists("/dev/shm" + name):
        os.unlink("/dev/shm" + name)                      # the killed sidecar's segment


# ---- H100 ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sidecar_scans_on_gpu_match_oracle(oracle_mod, tmp_path):
    """50 000 x 768 (>= 4096 rows: the tensor-core filter for L2 and cosine, the exact tiled kernel for manhattan), 16
    backend processes x 8 scans, LIMIT 10 and 64: identical to the oracle, and batched by the sidecar."""
    from pg_embedding_b200 import build, sidecar
    build.build()
    sidecar.client().pgemb_client_disconnect()
    name = f"/pgemb_gpu_scan_{os.getpid()}"
    srv = sidecar.SidecarProcess(name, slots=128, bulk_mb=16)
    srv.wait_ready(120)
    try:
        sidecar.connect(name)
        check_knn_seqscan(sidecar, oracle_mod)
        n, dims, P, per = 50_000, 768, 16, 8
        ks = [10 if p % 2 == 0 else 64 for p in range(P)]
        for mi, metric in enumerate(("l2", "cosine", "manhattan")):
            sub = tmp_path / metric
            sub.mkdir()
            check_concurrent_scans(sidecar, name, oracle_mod, metric, n, dims, ks, per, sub, rel_key=100 + mi)
    finally:
        sidecar.client().pgemb_client_disconnect()
        srv.stop()
