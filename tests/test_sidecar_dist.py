"""The SQL distance operators through pgemb_sidecar: `val <-> q`, `val <=> q`, `val <~> q` evaluated per row by the executor
(embedding.c:1022-1062) in the forked-backend deployment (DESIGN.md section 12, INTEGRATION.md sections 6-7).

Each backend process calls the reference-shaped hnsw_dist_func of libpgemb_client.so with one pair; the sidecar gathers the
calls pending at the same time per (metric, dim) into one pgemb_dist_batch call.  What must hold: every distance is the
oracle's (the compiled distfunc.c restatement) bit for bit, whatever the batch it was served in; concurrent calls share
pgemb_dist_batch calls; a bad request fails alone; searches and scans are served and counted as before; cancellation, a
killed backend and a dead sidecar behave as for every other request.

NaN results (cosine of a zero vector, overflowing magnitudes) are compared as NaN: the device's canonical NaN is not the
x86 default NaN of the CPU oracle, and the payload carries no distance.

CPU suite: the sidecar dlopen()s the host-emulated build of the C-ABI library (tests/emu).  `-m gpu`: the same through
the real libpgemb_b200.so on an H100, at 768 and 1536 dims with 64 backend processes."""
import json
import mmap
import os
import signal
import struct
import subprocess
import sys
import time

import numpy as np
import pytest

from test_sidecar_scan import Blocker, _slots_free, oracle_topk

pytestmark = pytest.mark.timeout(900, method="thread")
HERE = os.path.dirname(os.path.abspath(__file__))
EMU_ENV = {"PGEMB_EMU_SMS": "2", "PGEMB_EMU_TMA": "late"}
METRIC_NAMES = ("l2", "cosine", "manhattan")
PGEMB_ERR_ARG = 2
SLOT_FREE, SLOT_READY, SLOT_DONE, OP_DIST = 0, 2, 4, 13


def _start(lib, name, env=None, **kw):
    from pg_embedding_b200 import build, sidecar
    build.build_sidecar()
    srv = sidecar.SidecarProcess(name, lib=lib, env=env, **kw)
    srv.wait_ready(120)
    return srv


def _shm_name():
    return f"/pgemb_dist_{os.getpid()}_{int(time.time() * 1e3) % 100000}"


@pytest.fixture(scope="module")
def emulated_lib(tmp_path_factory):
    from emu_build import build_emulated
    return build_emulated(tmp_path_factory.mktemp("emu_sidecar_dist"))


def _serve(lib, env=None, **kw):
    """A sidecar (limits of the CPU suite unless overridden) with this process connected to it."""
    from pg_embedding_b200 import sidecar
    opts = dict(slots=32, max_dim=64, max_ef=64, bulk_mb=1, linger_us=20000)
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


# ---- pairs and the oracle --------------------------------------------------------------------------------------------
def _pairs(rng, n, dims, metrics=(0, 1, 2)):
    """n calls over the given dims and metrics: normal pairs plus zero vectors (cosine: NaN, distfunc.c:144), pairs of
    zero vectors, magnitudes whose squares overflow fp32, large finite magnitudes and tiny (subnormal-product) ones."""
    width = max(dims)
    metric = rng.choice(np.array(metrics), n)
    dim = rng.choice(np.array(dims), n)
    a = rng.standard_normal((n, width)).astype(np.float32)
    b = rng.standard_normal((n, width)).astype(np.float32)
    kind = rng.permutation(n) % 10
    a[kind == 1] = 0
    a[kind == 2] = 0
    b[kind == 2] = 0
    a[kind == 3] *= np.float32(1e20)
    a[kind == 4] *= np.float32(1e15)
    b[kind == 4] *= np.float32(3e14)
    b[kind == 5] *= np.float32(1e-21)
    return {"metric": metric.astype(np.int64), "dim": dim.astype(np.int64), "a": a, "b": b}


def oracle_dists(oracle_mod, c):
    """One oracle hnsw_dist_func per call: float32[n]."""
    return np.array([oracle_mod.dist("port", METRIC_NAMES[int(m)], c["a"][i, :d], c["b"][i, :d])
                     for i, (m, d) in enumerate(zip(c["metric"], c["dim"]))], np.float32)


def assert_bits(got_bits, want, what):
    """fp32 bits equal; NaN exactly where the oracle has NaN."""
    g = np.asarray(got_bits, np.uint32)
    w = np.asarray(want, np.float32)
    gn, wn = np.isnan(g.view(np.float32)), np.isnan(w)
    bad = np.flatnonzero((gn != wn) | (~gn & (g != w.view(np.uint32))))
    assert bad.size == 0, f"{what}: call {bad[0]}: got {g[bad[0]]:#010x}, oracle {w.view(np.uint32)[bad[0]]:#010x} ({bad.size} mismatches)"


# ---- the raw protocol (ipc.h) ----------------------------------------------------------------------------------------
class RawSegment:
    """Requests written straight into the segment: what a client without the library's own checks would send.  Only used
    while no other process claims slots (the backends of a test are parked at their start line), so plain stores in the
    protocol's order are enough."""

    VEC_OFF = 240                                                                     # pgemb_ipc_payload_vec_off()

    def __init__(self, name):
        self.f = open("/dev/shm" + name, "r+b")
        self.m = mmap.mmap(self.f.fileno(), 0)
        self.n_slots, self.max_dim, self.max_ef = struct.unpack_from("<III", self.m, 8)
        self.stride, self.slots_off = struct.unpack_from("<I", self.m, 20)[0], struct.unpack_from("<Q", self.m, 24)[0]
        self.labels_off = self.VEC_OFF + (2 * self.max_dim * 4 + 15) // 16 * 16
        self.dists_off = self.labels_off + self.max_ef * 8

    def _off(self, i):
        return self.slots_off + i * self.stride

    def submit(self, op, index_key=0, a=(0, 0, 0, 0), ef=0, vec=None):
        """Publish one request: op, index_key, a0..a3, ef and, unless None, `vec` (float32) at the start of the payload;
        returns its slot."""
        for i in range(self.n_slots):
            o = self._off(i)
            if struct.unpack_from("<I", self.m, o)[0] != SLOT_FREE:
                continue
            struct.pack_into("<IIii", self.m, o, 1, op, 0, os.getpid())             # CLAIMED, owner = this process
            struct.pack_into("<QQQQQ", self.m, o + 16, index_key, *a)                 # index_key, a0..a3
            struct.pack_into("<Ii", self.m, o + 56, ef, 0)
            struct.pack_into("<I", self.m, o + 64, 0)
            if vec is not None:
                v = np.ascontiguousarray(vec, np.float32).tobytes()
                self.m[o + self.VEC_OFF:o + self.VEC_OFF + len(v)] = v
            struct.pack_into("<I", self.m, o, SLOT_READY)
            return i
        raise AssertionError("no free slot")

    def submit_dist(self, dim, metric):
        """Publish one PGEMB_OP_DIST request (a0 = dim, a1 = metric, zero vectors); returns its slot."""
        return self.submit(OP_DIST, a=(dim, metric, 0, 0))

    def wait(self, i, timeout_s=60.0):
        """(status, message) of slot i once DONE; the slot is given back."""
        return self.wait_result(i, timeout_s)[:2]

    def wait_result(self, i, timeout_s=60.0):
        """(status, message, {"n_out", "a2", "labels", "dists"}) of slot i once DONE, the labels and distance bits of its
        first n_out results read as a search or scan result; the slot is given back."""
        o = self._off(i)
        deadline = time.time() + timeout_s
        while struct.unpack_from("<I", self.m, o)[0] != SLOT_DONE:
            assert time.time() < deadline, "raw request never completed"
            time.sleep(0.002)
        status = struct.unpack_from("<i", self.m, o + 8)[0]
        msg = bytes(self.m[o + 68:o + 68 + 164]).split(b"\0")[0].decode()
        n = struct.unpack_from("<i", self.m, o + 60)[0]
        k = max(0, min(n, self.max_ef))
        res = {"n_out": n, "a2": struct.unpack_from("<Q", self.m, o + 40)[0],
               "labels": list(struct.unpack_from(f"<{k}Q", self.m, o + self.labels_off)),
               "dists": list(struct.unpack_from(f"<{k}I", self.m, o + self.dists_off))}
        struct.pack_into("<i", self.m, o + 12, 0)                                     # FREE slots carry no pid
        struct.pack_into("<I", self.m, o, SLOT_FREE)
        return status, msg, res

    def close(self):
        self.m.close()
        self.f.close()


# ---- backend processes -----------------------------------------------------------------------------------------------
def _run_backends(shm, jobs, tmp_path, rel=None, blocker=None, before_go=None):
    """One backend process (tests/sidecar_dist_backend.py) per job (a dict of calls), all started together; with `blocker`
    (a function returning a Blocker), while the sidecar is busy, so that their first calls meet in one pass.  `rel`: the
    relation arguments of the interleaved search / scan / distance mode.  `before_go()` runs once the backends wait at
    their start line."""
    procs = []
    for p, calls in enumerate(jobs):
        cf, of = str(tmp_path / f"calls{p}.npz"), str(tmp_path / f"out{p}.json")
        np.savez(cf, **calls)
        cmd = [sys.executable, os.path.join(HERE, "sidecar_dist_backend.py"), shm, cf, of] + [str(r) for r in (rel or ())]
        procs.append((subprocess.Popen(cmd, stderr=subprocess.PIPE, text=True), of))
    deadline = time.time() + 300
    while not all(os.path.exists(of + ".ready") or pr.poll() is not None for pr, of in procs) and time.time() < deadline:
        time.sleep(0.01)
    if blocker is not None:
        blocker = blocker()
        blocker.wait_busy()
    if before_go is not None:
        before_go()
    open(str(tmp_path / "go"), "w").close()
    got = []
    for pr, of in procs:
        _, err = pr.communicate(timeout=600)
        assert pr.returncode == 0, err[-2000:]
        got.append(json.load(open(of)))
    if blocker is not None:
        blocker.join()
    return got


# ---- bodies shared by the CPU suite and -m gpu ---------------------------------------------------------------------------
def check_batched_dists(sc, name, oracle_mod, dims, P, per, tmp_path, blocker=None, seed=0):
    """P backend processes x `per` hnsw_dist_func calls over all metrics and `dims`: every result is the oracle's, the
    sidecar served them in fewer pgemb_dist_batch calls than pairs, and the search and scan counters did not move."""
    rng = np.random.default_rng([seed, P, per] + list(dims))
    jobs = [_pairs(rng, per, dims) for _ in range(P)]
    d0, s0, c0 = sc.dist_stats(), sc.stats(), sc.scan_stats()
    got = _run_backends(name, jobs, tmp_path, blocker=blocker)
    for p in range(P):
        assert_bits(got[p]["dist"], oracle_dists(oracle_mod, jobs[p]), f"backend {p}")
    d1 = sc.dist_stats()
    n_calls, n_dists = d1["calls"] - d0["calls"], d1["dists"] - d0["dists"]
    assert n_dists == P * per, (d0, d1)
    assert d1["max_batch"] > 1 and n_calls < n_dists, (d0, d1)                    # concurrent calls shared launches
    assert sc.stats() == s0 and sc.scan_stats() == c0
    return d1


# ---- CPU suite (emulated library) --------------------------------------------------------------------------------------
def test_concurrent_dists_are_batched_and_bit_exact(served, oracle_mod, tmp_path):
    """16 backend processes x 200 calls over l2 / cosine / manhattan at 3, 8, 13 and the sidecar's --max-dim (64), zero and
    extreme vectors included."""
    sc, name = served
    check_batched_dists(sc, name, oracle_mod, (3, 8, 13, 64), 16, 200, tmp_path, blocker=lambda: Blocker(sc, name, 900))


def test_mixed_groups_in_one_pass_and_bad_requests_fail_alone(served, oracle_mod, tmp_path):
    """Seven backends whose first call is pending in the same pass, over six (metric, dim) groups, next to raw requests
    with dim 0, dim beyond --max-dim and metric 3: one pgemb_dist_batch per group, each caller gets its own distance, and
    each bad request alone fails with PGEMB_ERR_ARG and the message of the one-pair path."""
    sc, name = served
    groups = [(0, 3), (0, 3), (1, 3), (0, 8), (2, 13), (1, 64), (2, 64)]
    rng = np.random.default_rng(7)
    jobs = []
    for m, d in groups:
        c = _pairs(rng, 1, (d,), (m,))
        c["a"][:], c["b"][:] = rng.standard_normal((2, 1, d)).astype(np.float32)     # no NaN: each result is a distance
        jobs.append(c)
    raw = RawSegment(name)
    bad = [(0, 0), (65, 0), (8, 3)]                                                   # (dim, metric)
    slots = []
    d0 = sc.dist_stats()
    try:
        got = _run_backends(name, jobs, tmp_path, blocker=lambda: Blocker(sc, name, 901),
                            before_go=lambda: slots.extend(raw.submit_dist(d, m) for d, m in bad))
        for (d, m), i in zip(bad, slots):
            assert raw.wait(i) == (PGEMB_ERR_ARG, "dist: bad dimension or metric"), (d, m)
    finally:
        raw.close()
    for p, c in enumerate(jobs):
        assert_bits(got[p]["dist"], oracle_dists(oracle_mod, c), f"group {groups[p]}")
    d1 = sc.dist_stats()
    assert d1["dists"] - d0["dists"] == len(groups), (d0, d1)
    assert d1["calls"] - d0["calls"] == len(set(groups)) and d1["max_batch"] == 2, (d0, d1)   # one call per group
    # through the library: metric 3 is not checked by the client, the sidecar refuses it; the NaN of a failed call
    import ctypes as C
    a = np.ones(4, np.float32)
    f32p = C.POINTER(C.c_float)
    assert np.isnan(sc.client().hnsw_dist_func(3, a.ctypes.data_as(f32p), a.ctypes.data_as(f32p), 4))
    assert sc.client().pgemb_client_last_error().decode() == "dist: bad dimension or metric"
    assert sc.dist("manhattan", a, 2 * a) == np.float32(4.0)
    assert _slots_free(name)


def test_dists_next_to_searches_and_scans(served, oracle_mod, tmp_path):
    """Four backends, each call one hnsw_search, one pgemb_client_scan_topk and one hnsw_dist_func: searches and scans are
    the oracle's, distances too, and each kind of request is counted by its own counters only."""
    sc, name = served
    rng = np.random.default_rng(23)
    n, dims, m, efc, ef, k = 300, 12, 4, 16, 12, 6
    x = rng.standard_normal((n, dims)).astype(np.float32)
    labels = np.arange(1000, 1000 + n, dtype=np.uint64)
    alive = np.arange(n) % 9 != 0
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, "l2", capacity=n)
    orc.build(x, labels)
    for i in np.flatnonzero(~alive):
        orc.mark_deleted(int(i))
    idx = sc.RemoteIndex(51, dims, m, efc, 64, "l2", capacity=n)
    idx.append_records(orc.records())
    P, per = 4, 5
    q = rng.standard_normal((P * per, dims)).astype(np.float32)
    jobs = []
    for p in range(P):
        c = _pairs(rng, per, (3, 8, 13, 64))
        c["q"] = q[p * per:(p + 1) * per]
        jobs.append(c)
    got = _run_backends(name, jobs, tmp_path, rel=(51, dims, m, efc, 64, "l2", ef, k))
    want_search = orc.search_many(q, ef)
    for p in range(P):
        assert_bits(got[p]["dist"], oracle_dists(oracle_mod, jobs[p]), f"backend {p}")
        for i in range(per):
            j = p * per + i
            assert got[p]["search"][i] == want_search["labels"][j, : want_search["n"][j]].tolist(), (p, i)
            assert got[p]["scan"][i] == oracle_topk(oracle_mod, "l2", x, labels, alive, q[j], k), (p, i)
    assert sc.stats()["searches"] == P * per and sc.scan_stats()["scans"] == P * per and sc.dist_stats()["dists"] == P * per
    idx.drop()


def test_cancelled_dist_returns_nan_and_the_sidecar_frees_its_slot(served, oracle_mod):
    """Query cancel while the call waits behind another backend's long request: hnsw_dist_func gives up with NaN, the
    sidecar later serves the abandoned pair, drops its result and frees the slot."""
    import ctypes as C
    sc, name = served
    a, b = np.arange(8, dtype=np.float32), np.ones(8, np.float32)
    blocker = Blocker(sc, name, 902)
    blocker.wait_busy()
    pending = C.c_int(1)
    cb = C.CFUNCTYPE(C.c_int)(lambda: pending.value)
    sc.client().pgemb_client_set_interrupt_check(C.cast(cb, C.c_void_p))
    try:
        t0 = time.time()
        assert np.isnan(sc.dist("l2", a, b))
        assert time.time() - t0 < 2.0
        assert "interrupted" in sc.client().pgemb_client_last_error().decode()
        pending.value = 0
    finally:
        sc.client().pgemb_client_set_interrupt_check(None)
    blocker.join()
    assert sc.dist("l2", a, b).tobytes() == oracle_mod.dist("port", "l2", a, b).tobytes()
    assert sc.dist_stats()["dists"] == 2                   # the abandoned pair was served, too
    assert _slots_free(name), "a slot was leaked"


def test_slot_of_a_backend_killed_while_its_dist_is_pending_is_reclaimed(served, oracle_mod, tmp_path):
    """A backend dies while its hnsw_dist_func request waits behind another backend's long request: the sidecar serves
    the orphaned request, its reclaim pass takes the slot back, and distances keep being served."""
    sc, name = served
    a, b = np.arange(8, dtype=np.float32), np.ones(8, np.float32)
    blocker = Blocker(sc, name, 903)
    blocker.wait_busy()
    cf, of = str(tmp_path / "calls.npz"), str(tmp_path / "out.json")
    np.savez(cf, metric=np.array([0]), dim=np.array([8]), a=a[None], b=b[None])
    open(str(tmp_path / "go"), "w").close()
    pr = subprocess.Popen([sys.executable, os.path.join(HERE, "sidecar_dist_backend.py"), name, cf, of], stderr=subprocess.PIPE, text=True)
    raw = RawSegment(name)
    try:
        deadline = time.time() + 60
        while not any(struct.unpack_from("<II", raw.m, raw._off(i)) == (SLOT_READY, OP_DIST) for i in range(raw.n_slots)):
            assert pr.poll() is None, pr.stderr.read()[-2000:]
            assert time.time() < deadline, "the backend's request never became pending"
            time.sleep(0.001)
    finally:
        raw.close()
    pr.send_signal(signal.SIGKILL)
    pr.wait()
    blocker.join()
    assert _slots_free(name, timeout_s=15.0), "the dead backend's slot was not reclaimed"
    assert sc.dist_stats()["dists"] == 1                   # the orphaned request was served
    assert sc.dist("l2", a, b).tobytes() == oracle_mod.dist("port", "l2", a, b).tobytes()


def test_dist_is_nan_when_the_sidecar_dies(emulated_lib, oracle_mod):
    from pg_embedding_b200 import sidecar
    name, srv = _serve(emulated_lib, env=EMU_ENV, slots=4, max_dim=16, max_ef=16)
    a, b = np.arange(8, dtype=np.float32), np.ones(8, np.float32)
    assert sidecar.dist("cosine", a, b).tobytes() == oracle_mod.dist("port", "cosine", a, b).tobytes()
    srv.proc.send_signal(signal.SIGKILL)
    srv.proc.wait()
    t0 = time.time()
    assert np.isnan(sidecar.dist("cosine", a, b))
    assert time.time() - t0 < 5.0
    sidecar.client().pgemb_client_disconnect()
    if os.path.exists("/dev/shm" + name):
        os.unlink("/dev/shm" + name)                      # the killed sidecar's segment


# ---- H100 ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dims", [768, 1536])
def test_sidecar_dists_on_gpu_match_oracle(oracle_mod, tmp_path, dims):
    """64 backend processes x 60 hnsw_dist_func calls over the three metrics through the real library: identical to the
    oracle, and batched by the sidecar."""
    from pg_embedding_b200 import build, sidecar
    build.build()
    sidecar.client().pgemb_client_disconnect()
    name = f"/pgemb_gpu_dist_{os.getpid()}_{dims}"
    srv = sidecar.SidecarProcess(name, slots=128, bulk_mb=1)
    srv.wait_ready(120)
    try:
        sidecar.connect(name)
        check_batched_dists(sidecar, name, oracle_mod, (dims,), 64, 60, tmp_path, seed=dims)
    finally:
        sidecar.client().pgemb_client_disconnect()
        srv.stop()
