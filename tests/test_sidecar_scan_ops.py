"""The index-less scan through pgemb_sidecar under any of the three operators: `ORDER BY val <op> q LIMIT k` without the
index where <op> need not be the relation's opclass operator (pgemb_client_scan_topk_op).

Backend processes scan one relation with <->, <=>, <~> and the opclass's own operator (pgemb_client_scan_topk, which sends
metric code 0) mixed.  What must hold: every answer is the oracle's (hnsw_dist_func of the query's operator per row, live
rows sorted by (dist, label), labels and distance bits); the scans pending together are served by one pgemb_scan_topk_op
call per (relation, metric, k), a scan of the relation's own operator sharing the call of the scans that name it; a bad
metric is refused by the client before anything is sent and by the sidecar for its group alone.

CPU suite: the sidecar dlopen()s the host-emulated build of the C-ABI library (tests/emu).  The 16-backend run on the H100
is tests/test_gpu_scan_ops.py."""
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np
import pytest

import test_sidecar_scan as T

pytestmark = pytest.mark.timeout(900, method="thread")
HERE = os.path.dirname(os.path.abspath(__file__))
OPS = ("own", "l2", "cosine", "manhattan")
PGEMB_OP_SCAN, PGEMB_OP_BUILD, SLOT_READY, SLOT_BUSY, SLOT_DONE = 15, 12, 2, 3, 4
PGEMB_ERR_ARG = 2


@pytest.fixture(scope="module")
def emulated_lib(tmp_path_factory):
    from emu_build import build_emulated
    return build_emulated(tmp_path_factory.mktemp("emu_sidecar_scan_ops"))


@pytest.fixture()
def served(emulated_lib):
    from pg_embedding_b200 import sidecar
    name, srv = T._serve(emulated_lib, env=T.EMU_ENV)
    yield sidecar, name
    T._stop(srv)


# ---- the shared-memory segment, read (and for one raw request written) by the test ------------------------------------
def _segment(name):
    raw = bytearray(open("/dev/shm" + name, "rb").read())
    n_slots, stride, slots_off = struct.unpack_from("<I", raw, 8)[0], struct.unpack_from("<I", raw, 20)[0], struct.unpack_from("<Q", raw, 24)[0]
    return raw, n_slots, stride, slots_off


def _slot_states(name):
    """(state, op) of every slot."""
    raw, n_slots, stride, slots_off = _segment(name)
    return [struct.unpack_from("<II", raw, slots_off + i * stride) for i in range(n_slots)]


class RawScan:
    """A PGEMB_OP_SCAN request written straight into a FREE slot (ipc.h's PgembIpcSlot), with a metric code no client library
    sends: the sidecar's own check of the code.  Only written while no other process claims slots."""
    VEC_OFF = 240      # (sizeof(PgembIpcSlot) = 232, rounded up to 16)

    def __init__(self, name, rel_key, k, metric_code, q):
        import mmap
        self.fd = os.open("/dev/shm" + name, os.O_RDWR)
        self.mm = mmap.mmap(self.fd, 0)
        _, n_slots, stride, slots_off = _segment(name)
        free = [i for i, (stt, _) in enumerate(_slot_states(name)) if stt == 0]
        self.off = slots_off + free[-1] * stride
        struct.pack_into("<IiiQQQQQIiI", self.mm, self.off + 4, PGEMB_OP_SCAN, 0, os.getpid(), rel_key, k, metric_code, 0, 0, 0, 0, 0)
        self.mm[self.off + self.VEC_OFF:self.off + self.VEC_OFF + q.size * 4] = np.ascontiguousarray(q, np.float32).tobytes()
        struct.pack_into("<I", self.mm, self.off, SLOT_READY)       # publish last

    def result(self, timeout_s=120.0):
        """(status, message) once the sidecar is done with it; frees the slot."""
        deadline = time.time() + timeout_s
        while struct.unpack_from("<I", self.mm, self.off)[0] != SLOT_DONE:
            assert time.time() < deadline, "the sidecar never answered the raw request"
            time.sleep(0.005)
        status = struct.unpack_from("<i", self.mm, self.off + 8)[0]
        err = bytes(self.mm[self.off + 68:self.off + 68 + 164]).split(b"\0")[0].decode()
        struct.pack_into("<i", self.mm, self.off + 12, 0)
        struct.pack_into("<I", self.mm, self.off, 0)
        self.mm.close()
        os.close(self.fd)
        return status, err


# ---- backend processes -------------------------------------------------------------------------------------------------
def _run_backends(shm, rel_key, cfg, jobs, tmp_path, blocker=None, before_go=None, during=None):
    """One backend process per job (op, k, queries), all started together; with `blocker` (a function returning a
    T.Blocker), while the sidecar is busy.  before_go() runs once the backends wait at the start line, during() while they
    run."""
    procs = []
    for p, (op, k, q) in enumerate(jobs):
        qf, of = str(tmp_path / f"q{p}.npy"), str(tmp_path / f"out{p}.json")
        np.save(qf, q)
        cmd = [sys.executable, os.path.join(HERE, "sidecar_scan_op_backend.py"), shm, str(rel_key)] + [str(c) for c in cfg] + [op, str(k), qf, of]
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


def _all_queued_behind_the_build(name, want, timeout_s=60.0):
    """Wait until `want` scans are READY while the blocker's build is still running: then the sidecar collects all of them
    in its next pass.  Returns whether that was seen."""
    deadline = time.time() + timeout_s
    while time.time() < deadline:
        st = _slot_states(name)
        ready = sum(1 for s in st if s == (SLOT_READY, PGEMB_OP_SCAN))
        building = any(s == (SLOT_BUSY, PGEMB_OP_BUILD) for s in st)
        if ready == want and building:
            return True
        if not building:
            return False
        time.sleep(0.001)
    return False


def check_mixed_operator_scans(sc, name, oracle_mod, mirror, n, dims, P, per, tmp_path, ks=(5, 9), rel_key=61, blocker=False, bad_code=None):
    """P backends x `per` scans of one relation (opclass `mirror`); backend p uses operator OPS[p % 4] and LIMIT
    ks[(p // 4) % len(ks)].  Every answer is the oracle's and the search counters do not move.  With `blocker` the first scan
    of every backend is queued behind a long request, so that with per = 1 the sidecar serves them all in one pass: exactly
    one call per (metric, k) group.  `bad_code`: a raw request with that metric code joins the pass and fails alone."""
    rng = np.random.default_rng([n, dims, OPS.index(mirror) if mirror in OPS else 0])
    x, labels, alive = T._table(rng, n, dims, mirror)
    idx = T._mirror(sc, rel_key, x, labels, alive, mirror)
    q = rng.standard_normal((P * per, dims)).astype(np.float32)
    jobs = [(OPS[p % 4], ks[(p // 4) % len(ks)], q[p * per:(p + 1) * per]) for p in range(P)]
    resolved = [(mirror if op == "own" else op, k) for op, k, _ in jobs]
    s0, c0 = sc.stats(), sc.scan_stats()
    raw, seen = [], []
    before_go = (lambda: raw.append(RawScan(name, rel_key, 4, bad_code, q[0]))) if bad_code is not None else None
    during = (lambda: seen.append(_all_queued_behind_the_build(name, P + len(raw)))) if blocker else None
    got = _run_backends(name, rel_key, (dims, 3, 8, 16, mirror), jobs, tmp_path, blocker=(lambda: T.Blocker(sc, name, 903)) if blocker else None,
                        before_go=before_go, during=during)
    for p, (metric, k) in enumerate(resolved):
        for i in range(per):
            assert got[p][i] == T.oracle_topk(oracle_mod, metric, x, labels, alive, q[p * per + i], k), (mirror, jobs[p][0], k, p, i)
    c1 = sc.scan_stats()
    assert c1["scans"] - c0["scans"] == P * per, (c0, c1)
    if blocker and per == 1:
        assert seen == [True], "the backends' scans did not all queue up behind the blocking build"
        assert c1["calls"] - c0["calls"] == len(set(resolved)), (resolved, c0, c1)
    else:
        assert c1["calls"] - c0["calls"] < P * per and c1["max_batch"] >= 2, (c0, c1)
    if raw:
        status, err = raw[0].result()
        assert status == PGEMB_ERR_ARG and "unknown distance function" in err, (status, err)
    s1 = sc.stats()
    assert (s1["batches"], s1["searches"]) == (s0["batches"], s0["searches"]), (s0, s1)
    idx.drop()


# ---- CPU suite (emulated library) --------------------------------------------------------------------------------------
@pytest.mark.parametrize("mirror", ["l2", "cosine", "manhattan"])
def test_mixed_operator_scans_get_the_oracle_results(served, oracle_mod, mirror, tmp_path):
    """8 backends x 4 scans on one relation: the four operators (the opclass's own twice over) at LIMIT 5 and 9."""
    sc, name = served
    check_mixed_operator_scans(sc, name, oracle_mod, mirror, 300, 16, 8, 4, tmp_path, blocker=True)


def test_one_call_per_relation_metric_and_k(served, oracle_mod, tmp_path):
    """8 backends' scans queued together behind a long request on an ann_l2_ops relation: <-> and the opclass's own operator
    at LIMIT 5 share one call; <=> and <~> get one each; LIMIT 9 the same again -- 6 calls for 8 scans.  A raw request with
    an unknown metric code in the same pass fails with PGEMB_ERR_ARG and leaves the other groups alone."""
    sc, name = served
    check_mixed_operator_scans(sc, name, oracle_mod, "l2", 300, 16, 8, 1, tmp_path, blocker=True, bad_code=7)
    assert T._slots_free(name)


@pytest.mark.parametrize("metric_code", [0, 2])
def test_scan_without_a_metric_still_takes_the_relations_own(served, oracle_mod, metric_code):
    """The old request (metric field 0, pgemb_client_scan_topk) and the new one naming the opclass's operator both get the
    relation's own operator: the same bytes as before.  (Code 2 = <=> on an ann_cos_ops relation.)"""
    sc, name = served
    rng = np.random.default_rng(9)
    x, labels, alive = T._table(rng, 120, 8, "cosine")
    idx = T._mirror(sc, 71, x, labels, alive, "cosine")
    q = rng.standard_normal(8).astype(np.float32)
    want = T.oracle_topk(oracle_mod, "cosine", x, labels, alive, q, 7)
    assert T._row(idx.scan_topk(q, 7, metric=None if metric_code == 0 else metric_code - 1)) == want
    assert T._row(idx.scan_topk(q, 7, metric="cosine")) == want
    assert T._row(idx.scan_topk(q, 7)) == want
    assert T._slots_free(name)
    idx.drop()


def test_bad_metric_is_refused_before_anything_is_sent(served, oracle_mod):
    sc, name = served
    rng = np.random.default_rng(10)
    x, labels, alive = T._table(rng, 60, 8, "l2")
    idx = T._mirror(sc, 72, x, labels, alive, "l2")
    for bad in (-1, 3, 1 << 20):
        with pytest.raises(sc.SidecarError, match=f"pgemb status {PGEMB_ERR_ARG}: pgemb_client_scan_topk_op: unknown distance function"):
            idx.scan_topk(x[0], 4, metric=bad)
    with pytest.raises(KeyError):
        idx.scan_topk(x[0], 4, metric="hamming")
    with pytest.raises(sc.SidecarError, match=f"pgemb status {PGEMB_ERR_ARG}: pgemb_client_scan_topk_op: k = 0 outside"):
        idx.scan_topk(x[0], 0, metric="manhattan")
    assert sc.scan_stats()["scans"] == 0
    assert T._row(idx.scan_topk(x[1], 4, metric="manhattan")) == T.oracle_topk(oracle_mod, "manhattan", x, labels, alive, x[1], 4)
    assert T._slots_free(name)
    idx.drop()
