"""The sidecar's checks on a batched group -- searches per (relation, ef), scans per (relation, k), distances per (metric,
dim) -- for requests the client library refuses before it claims a slot, so that only a client without its checks can
send them (tests/test_sidecar_dist.py RawSegment).  Published in one pass next to a valid group of each kind: each bad
request fails alone, with PGEMB_ERR_ARG and its message, the valid groups get the oracle's results, and each kind's
counters move by exactly its own group."""
import numpy as np
import pytest

from test_sidecar_dist import PGEMB_ERR_ARG, OP_DIST, RawSegment, emulated_lib, served  # noqa: F401 (fixtures)
from test_sidecar_scan import Blocker, _slots_free, oracle_topk

pytestmark = pytest.mark.timeout(900, method="thread")
OP_SEARCH, OP_SCAN = 4, 15
NO_INDEX = "no device index attached for this relation key"


def test_bad_batched_requests_fail_alone_next_to_valid_groups(served, oracle_mod):
    sc, name = served
    rng = np.random.default_rng(31)
    n, dims, m, efc, ef, k, rel = 200, 12, 4, 16, 12, 6, 61
    x = rng.standard_normal((n, dims)).astype(np.float32)
    labels = np.arange(5000, 5000 + n, dtype=np.uint64)
    alive = np.arange(n) % 7 != 0
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, "l2", capacity=n)
    orc.build(x, labels)
    for i in np.flatnonzero(~alive):
        orc.mark_deleted(int(i))
    idx = sc.RemoteIndex(rel, dims, m, efc, 64, "l2", capacity=n)
    idx.append_records(orc.records())
    q = rng.standard_normal((6, dims)).astype(np.float32)
    pairs = rng.standard_normal((3, 2, 8)).astype(np.float32)
    raw = RawSegment(name)
    max_ef = raw.max_ef                                                   # 64: the scan limit min(4096, --max-ef) too
    bad = [(OP_SEARCH, rel, 0, 0, "efSearch outside the sidecar's --max-ef"),
           (OP_SEARCH, rel, 0, max_ef + 1, "efSearch outside the sidecar's --max-ef"),
           (OP_SEARCH, 999, 0, ef, NO_INDEX),
           (OP_SCAN, rel, 0, 0, "scan: k outside 1 .. min(4096, the sidecar's --max-ef)"),
           (OP_SCAN, rel, max_ef + 1, 0, "scan: k outside 1 .. min(4096, the sidecar's --max-ef)"),
           (OP_SCAN, 999, k, 0, NO_INDEX)]                                # (op, relation, a0 = k, ef, message)
    s0, c0, d0 = sc.stats(), sc.scan_stats(), sc.dist_stats()
    blocker = Blocker(sc, name, 904)
    try:
        blocker.wait_busy()
        searches = [raw.submit(OP_SEARCH, rel, ef=ef, vec=q[i]) for i in range(3)]
        scans = [raw.submit(OP_SCAN, rel, a=(k, 0, 0, 0), vec=q[3 + i]) for i in range(3)]
        dists = []
        for a, b in pairs:
            v = np.zeros(2 * raw.max_dim, np.float32)
            v[:8], v[raw.max_dim:raw.max_dim + 8] = a, b
            dists.append(raw.submit(OP_DIST, a=(8, 0, 0, 0), vec=v))
        bad_slots = [raw.submit(op, key, a=(a0, 0, 0, 0), ef=e, vec=q[0]) for op, key, a0, e, _ in bad]
        blocker.join()
        for (op, key, a0, e, msg), i in zip(bad, bad_slots):
            assert raw.wait(i) == (PGEMB_ERR_ARG, msg), (op, key, a0, e)
        got_search = [raw.wait_result(i) for i in searches]
        got_scan = [raw.wait_result(i) for i in scans]
        got_dist = [raw.wait_result(i) for i in dists]
    finally:
        raw.close()
    want_search = orc.search_many(q[:3], ef)
    for i, (status, msg, r) in enumerate(got_search):
        assert (status, msg) == (0, ""), msg
        assert r["labels"] == want_search["labels"][i, : want_search["n"][i]].tolist(), i
    for i, (status, msg, r) in enumerate(got_scan):
        assert (status, msg) == (0, ""), msg
        assert {"labels": r["labels"], "dists": r["dists"]} == oracle_topk(oracle_mod, "l2", x, labels, alive, q[3 + i], k), i
    for (a, b), (status, msg, r) in zip(pairs, got_dist):
        assert (status, msg) == (0, ""), msg
        assert r["a2"] == int(oracle_mod.dist("port", "l2", a, b).view(np.uint32))
    s1, c1, d1 = sc.stats(), sc.scan_stats(), sc.dist_stats()
    assert (s1["batches"] - s0["batches"], s1["searches"] - s0["searches"], s1["max_batch"]) == (1, 3, 3), (s0, s1)
    assert (c1["calls"] - c0["calls"], c1["scans"] - c0["scans"], c1["max_batch"]) == (1, 3, 3), (c0, c1)
    assert (d1["calls"] - d0["calls"], d1["dists"] - d0["dists"], d1["max_batch"]) == (1, 3, 3), (d0, d1)
    assert _slots_free(name)
    idx.drop()
