"""The exact scan under any of the three operators over a mirror of any metric (pgemb_scan_topk_op): `ORDER BY val <op> q
LIMIT k` without the index when <op> is not the opclass's, e.g. a relation indexed with ann_l2_ops queried with <=> or <~>.

For each of the 3 x 3 (mirror metric, query metric) pairs the result must be the oracle's -- hnsw_dist_func(query metric)
per row, live rows sorted by (dist, label), labels and distance bits -- on the tensor-core filter (L2, cosine) and on the
exact kernels alike, with no tripwire fallback.  A cosine or L2 scan over a mirror that has no row norms yet computes them
first.

tests/test_scan_ops_emulated.py runs the same bodies on the host-emulated library at small sizes."""
import ctypes as C

import numpy as np
import pytest

METRICS = ("l2", "cosine", "manhattan")
PAIRS = [(m, q) for m in METRICS for q in METRICS]
DELETED = np.uint64(1 << 48)


@pytest.fixture(scope="module")
def pg():
    import pg_embedding_b200 as pg
    from pg_embedding_b200 import build
    build.build()
    if pg.device_count() < 1:
        pytest.fail("no CUDA device: the product path has no CPU fallback")
    return pg


def counters():
    from pg_embedding_b200 import _lib
    out = (C.c_uint64 * 6)()
    _lib.load().pgemb_scan_counters(out)
    return dict(tc=out[0], pairs=out[1], rescored=out[2], fallbacks=out[3], overflow=out[4], exact=out[5])


def delta(c0, c1):
    return {k: c1[k] - c0[k] for k in c0}


def oracle_topk(oracle_mod, metric, x, labels, q, k):
    """hnsw_dist_func(metric) per row (the oracle's restatement), live rows sorted by (dist, label) in the scan's order of the
    fp32 bit patterns (NaN after +inf): labels and distance bits."""
    d = np.asarray(oracle_mod.dist_many("port", metric, q, x), np.float32)
    b = d.view(np.uint32)
    key = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000))
    order = np.lexsort((labels, key))
    order = order[((labels[order] >> np.uint64(48)) & np.uint64(1)) == 0][:k]
    return labels[order].tolist(), d[order].view(np.uint32).tolist()


def assert_oracle(oracle_mod, metric, x, labels, q, k, got, rows, what):
    for i in rows:
        want_l, want_d = oracle_topk(oracle_mod, metric, x, labels, q[i], k)
        n = int(got["n"][i])
        assert n == len(want_l), (what, i)
        assert got["labels"][i, :n].tolist() == want_l, (what, i)
        assert got["dists"][i, :n].view(np.uint32).tolist() == want_d, (what, i)
        assert (got["labels"][i, n:] == np.uint64(0xFFFFFFFFFFFFFFFF)).all() and np.isinf(got["dists"][i, n:]).all(), (what, i)


def table(rng, n, dims, nq):
    """Clustered rows (so the filter has something to discard) with an exact duplicate (a tie broken by label), a zero row
    (cosine NaN), every 11th row deleted; queries near the clusters, one of them the zero vector, one equal to a row."""
    c = rng.standard_normal((12, dims)).astype(np.float32)
    x = (c[rng.integers(0, 12, n)] + 0.15 * rng.standard_normal((n, dims))).astype(np.float32) + np.float32(0.5)
    q = (c[rng.integers(0, 12, nq)] + 0.15 * rng.standard_normal((nq, dims))).astype(np.float32) + np.float32(0.5)
    x[n // 2] = x[n // 3]
    x[n // 4] = 0.0
    q[1] = 0.0
    q[2] = x[n // 5]
    labels = rng.permutation(n).astype(np.uint64) + np.uint64(3)
    labels[::11] |= DELETED
    return x, q, labels


def check_pairs(pg, oracle_mod, monkeypatch, n, dims, nq, k, oracle_rows):
    """The nine (mirror, query) metric pairs: PGEMB_SCAN_TC=2 (the tensor-core filter for L2 / cosine queries) and =0 give the
    same bytes, equal to the oracle's, and the filter never falls back.  A query of the mirror's own metric gives
    pgemb_scan_topk's bytes."""
    rng = np.random.default_rng([n, dims, nq])
    x, q, labels = table(rng, n, dims, nq)
    for mirror in METRICS:
        idx = pg.HnswIndex(dims, 4, 8, 16, mirror, capacity=n)
        idx.append(x, labels)
        for metric in METRICS:
            monkeypatch.setenv("PGEMB_SCAN_TC", "2")
            c0 = counters()
            got = idx.scan_topk(q, k, metric=metric)
            d = delta(c0, counters())
            assert d["fallbacks"] == 0, (mirror, metric, "the TF32 error bound was exceeded (tripwire)")
            if metric == "manhattan":
                assert (d["tc"], d["exact"]) == (0, 1), (mirror, metric, d)
            else:
                assert (d["tc"], d["exact"], d["pairs"]) == (1, 0, nq * n), (mirror, metric, d)
            monkeypatch.setenv("PGEMB_SCAN_TC", "0")
            want = idx.scan_topk(q, k, metric=metric)
            for f in ("labels", "dists", "n"):
                assert got[f].tobytes() == want[f].tobytes(), (mirror, metric, f)
            assert_oracle(oracle_mod, metric, x, labels, q, k, got, oracle_rows, (mirror, metric))
            if metric == mirror:
                for tc in ("0", "2"):
                    monkeypatch.setenv("PGEMB_SCAN_TC", tc)
                    own, named = idx.scan_topk(q, k), idx.scan_topk(q, k, metric=metric)
                    for f in ("labels", "dists", "n"):
                        assert own[f].tobytes() == named[f].tobytes(), (mirror, tc, f)
        idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dims", [768, 99], ids=["d768", "d99"])
def test_scan_ops_nine_pairs(pg, oracle_mod, monkeypatch, dims):
    """50 000 rows, 64 queries, k 10; 99 dims is neither a multiple of the 32-float k-block nor of the 4-float row unit."""
    check_pairs(pg, oracle_mod, monkeypatch, 50_000, dims, 64, 10, range(0, 64, 7))


def check_norms_on_demand(pg, oracle_mod, monkeypatch, n, dims, nq, k, tc_first):
    """An L2 mirror has no row norms until a scan needs them: a cosine scan first (exact kernels or the filter, `tc_first`),
    then L2, then rows appended and cosine again -- every answer the oracle's and equal to a fresh mirror's."""
    rng = np.random.default_rng([n, dims, 7])
    x, q, labels = table(rng, n, dims, nq)
    first = n * 3 // 4
    idx = pg.HnswIndex(dims, 4, 8, 16, "l2", capacity=n)
    idx.append(x[:first], labels[:first])
    monkeypatch.setenv("PGEMB_SCAN_TC", tc_first)
    steps = [("cosine", first), ("l2", first), ("cosine", n)]
    for metric, rows in steps:
        if rows > len(idx):
            idx.append(x[len(idx):rows], labels[len(idx):rows])
        got = idx.scan_topk(q, k, metric=metric)
        assert_oracle(oracle_mod, metric, x[:rows], labels[:rows], q, k, got, range(nq), (tc_first, metric, rows))
        monkeypatch.setenv("PGEMB_SCAN_TC", "2")
    fresh = pg.HnswIndex(dims, 4, 8, 16, "cosine", capacity=n)
    fresh.append(x, labels)
    for tc in ("0", "2"):
        monkeypatch.setenv("PGEMB_SCAN_TC", tc)
        a, b = idx.scan_topk(q, k, metric="cosine"), fresh.scan_topk(q, k)
        for f in ("labels", "dists", "n"):
            assert a[f].tobytes() == b[f].tobytes(), (tc, f)
    idx.close()
    fresh.close()


@pytest.mark.gpu
@pytest.mark.parametrize("tc_first", ["0", "2"])
def test_scan_ops_l2_mirror_norms_on_demand(pg, oracle_mod, monkeypatch, tc_first):
    check_norms_on_demand(pg, oracle_mod, monkeypatch, 20_000, 200, 16, 8, tc_first)


@pytest.mark.gpu
def test_scan_ops_device_entry_point(pg, monkeypatch):
    """pgemb_scan_topk_op_device with device pointers == pgemb_scan_topk_op, byte for byte, and a bad metric is refused."""
    import torch
    from pg_embedding_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(4)
    n, dims, nq, k = 9000, 64, 20, 12
    x, q, labels = table(rng, n, dims, nq)
    idx = pg.HnswIndex(dims, 4, 8, 16, "manhattan", capacity=n)
    idx.append(x, labels)
    monkeypatch.delenv("PGEMB_SCAN_TC", raising=False)
    for mi, metric in enumerate(METRICS):
        tq = torch.from_numpy(q).cuda()
        tl = torch.zeros((nq, k), dtype=torch.int64, device="cuda")
        td = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
        tn = torch.zeros(nq, dtype=torch.int32, device="cuda")
        _lib.check(lib.pgemb_scan_topk_op_device(idx.dev, mi, nq, tq.data_ptr(), k, tl.data_ptr(), td.data_ptr(), tn.data_ptr(), None))
        host = idx.scan_topk(q, k, metric=metric)
        assert tl.cpu().numpy().view(np.uint64).tobytes() == host["labels"].tobytes()
        assert td.cpu().numpy().tobytes() == host["dists"].tobytes() and tn.cpu().numpy().tolist() == host["n"].tolist()
    for bad in (-1, 3):
        assert lib.pgemb_scan_topk_op_device(idx.dev, bad, nq, tq.data_ptr(), k, tl.data_ptr(), None, tn.data_ptr(), None) == 2
    idx.close()


@pytest.mark.gpu
def test_sidecar_mixed_operator_scans_on_gpu(oracle_mod, tmp_path):
    """16 backend processes scan one 50 000 x 768 relation (ann_l2_ops) with <->, <=>, <~> and the opclass's own operator
    mixed: every answer is the oracle's, and concurrent scans of one (metric, k) share a pgemb_scan_topk_op call."""
    import test_sidecar_scan as T
    import test_sidecar_scan_ops as S
    from pg_embedding_b200 import build, sidecar
    build.build()
    name, srv = T._serve(None, slots=128, bulk_mb=64, max_ef=1024, max_dim=2000, linger_us=None)
    try:
        S.check_mixed_operator_scans(sidecar, name, oracle_mod, "l2", 50_000, 768, 16, 6, tmp_path, ks=(10, 64))
    finally:
        T._stop(srv)
