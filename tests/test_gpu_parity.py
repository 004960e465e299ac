"""GPU parity tests proper: the CUDA path, called through the C ABI, against the CPU oracle on the same
seeded inputs.  Bar: bit-exact ids / labels / link lists AND bit-exact fp32 distances (tolerance 0 --
north_star allows 1e-5 relative, the kernels reproduce the reference's summation order exactly).

The checker is the C restatement (`port`, buildable on the GPU box) and, when the prebuilt
oracle/_ref/libpgemb_ref.so travelled with the tree, the compiled reference itself (`ref`)."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

METRICS = ["l2", "cosine", "manhattan"]


@pytest.fixture(scope="module")
def pg():
    import pg_embedding_b200 as pg
    from pg_embedding_b200 import build
    build.build()
    if pg.device_count() < 1:
        pytest.fail("no CUDA device: the product path has no CPU fallback")
    return pg


class kernel_mode:
    """Pin the traversal kernel variant: "1" = latency mode (a CTA per query, used by default below one query per
    SM), "0" = throughput mode (a warp per query).  Both must give the reference's results."""

    def __init__(self, coop):
        self.coop = coop

    def __enter__(self):
        self.old = os.environ.get("PGEMB_COOP")
        os.environ["PGEMB_COOP"] = self.coop

    def __exit__(self, *a):
        if self.old is None:
            os.environ.pop("PGEMB_COOP", None)
        else:
            os.environ["PGEMB_COOP"] = self.old


def checkers(oracle_mod):
    return ["port"] + (["ref"] if oracle_mod.available("ref") else [])


def _data(rng, n, dim, clustered=True, dup_frac=0.0, levels=0):
    if levels:
        x = rng.integers(0, levels, size=(n, dim)).astype(np.float32)
    elif clustered:
        c = rng.standard_normal((max(4, int(np.sqrt(n))), dim)).astype(np.float32)
        x = c[rng.integers(0, len(c), n)] + 0.3 * rng.standard_normal((n, dim)).astype(np.float32)
    else:
        x = rng.standard_normal((n, dim)).astype(np.float32)
    if dup_frac > 0:
        k = int(n * dup_frac)
        x[rng.integers(0, n, k)] = x[rng.integers(0, n, k)]
    return np.ascontiguousarray(x, dtype=np.float32)


# ---------------------------------------------------------------------------------------------------
# a1-a4: distances
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_distance_bits(pg, oracle_mod, metric):
    rng = np.random.default_rng(11)
    dims = list(range(1, 40)) + [63, 64, 65, 100, 127, 128, 129, 300, 768, 769, 1536, 2000]
    for dim in dims:
        a = rng.standard_normal((48, dim)).astype(np.float32) * rng.choice([1e-3, 1.0, 37.0], size=(48, 1)).astype(np.float32)
        b = rng.standard_normal((48, dim)).astype(np.float32)
        got = pg.dist_batch(metric, a, b)
        for which in checkers(oracle_mod):
            want = oracle_mod.dist_many(which, metric, a, b)
            assert got.tobytes() == want.tobytes(), (metric, dim, which, np.flatnonzero(got != want)[:4])
        got = pg.dist_batch(metric, a[0], b)
        want = oracle_mod.dist_many("port", metric, a[0], b)
        assert got.tobytes() == want.tobytes(), (metric, dim, "broadcast")


def test_sql_distance_functions(pg, oracle_mod):
    a, b = np.array([0, 1, 2], np.float32), np.array([3, 3, 3], np.float32)
    assert pg.l2_distance(a, b) == oracle_mod.dist("port", "l2", a, b)
    assert pg.cosine_distance(a, b) == oracle_mod.dist("port", "cosine", a, b)
    assert pg.manhattan_distance(a, b) == np.float32(6.0)
    with pytest.raises(ValueError, match="different array dimensions 3 and 2"):  # embedding.c:1031-1035
        pg.l2_distance(a, b[:2])


# ---------------------------------------------------------------------------------------------------
# golden KATs (reference pg_regress expected outputs) through the reference-shaped entry points
# ---------------------------------------------------------------------------------------------------
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "kat_regress.json")))["cases"]


def tid_label(blk, pos, flags=0):
    return (blk >> 16) | ((blk & 0xFFFF) << 16) | (pos << 32) | (flags << 48)


@pytest.mark.parametrize("case", GOLD, ids=[c["name"] for c in GOLD])
def test_kat_regress(pg, case):
    o = case["options"]
    for metric in case.get("expected", case.get("expected_tids")).keys():
        idx = pg.HnswIndex(o["dims"], o["m"], o["efconstruction"], o["efsearch"], metric, capacity=64)
        by_label = {}
        for r in case.get("rows_before_truncate", []):
            idx.insert(np.array(r["val"], np.float32), tid_label(*r["tid"]))
        if "rows_before_truncate" in case:
            idx.truncate()
        for r in case["rows"]:
            lab = tid_label(*r["tid"])
            idx.insert(np.array(r["val"], np.float32), lab)
            by_label[lab] = r
        if "delete_all_then_insert" in case:
            idx.mark_deleted(np.arange(len(idx)))
            by_label = {}
            for r in case["delete_all_then_insert"]:
                lab = tid_label(*r["tid"])
                idx.insert(np.array(r["val"], np.float32), lab)
                by_label[lab] = r
        labels = idx.search(np.array(case["query"], np.float32))  # hnsw_search
        rows = [by_label[int(l)] for l in labels]
        if "expected" in case:
            assert [r["val"] for r in rows] == case["expected"][metric], metric
        if "expected_tids" in case:
            assert [r["tid"] for r in rows] == case["expected_tids"][metric], metric
        if "expected_distances" in case:
            out = idx.search_batch(np.array([case["query"]], np.float32))
            np.testing.assert_allclose(out["dists"][0, : out["n"][0]], case["expected_distances"][metric], rtol=0, atol=5e-7)
        idx.close()


# ---------------------------------------------------------------------------------------------------
# a6-a8: search on an identical graph
# ---------------------------------------------------------------------------------------------------
SEARCH_CFGS = [
    # dims, m, efC, n, kwargs for _data, efs
    (3, 3, 16, 300, dict(levels=3), (1, 2, 5, 64)),                 # tie-heavy: overflow machinery
    (2, 3, 8, 400, dict(levels=2), (1, 3, 16)),                     # massive duplicates
    (16, 8, 40, 2000, dict(), (1, 10, 64, 100)),
    (33, 5, 20, 1000, dict(dup_frac=0.1), (7, 64)),                 # dims % 4 != 0 (row padding, scalar tails)
    (128, 16, 64, 3000, dict(), (64, 200)),                         # BASELINE configs[1] shape (small N)
    (100, 20, 32, 1500, dict(), (64,)),                             # maxM = 40 > one warp chunk
    (24, 100, 16, 700, dict(), (64,)),                              # reference defaults m=100 -> maxM=200
    (768, 32, 48, 600, dict(), (64,)),                              # north-star row shape
]


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("cfg", SEARCH_CFGS, ids=[f"d{c[0]}m{c[1]}n{c[3]}" for c in SEARCH_CFGS])
def test_search_identical_to_oracle(pg, oracle_mod, metric, cfg):
    dims, m, efc, n, kw, efs = cfg
    rng = np.random.default_rng(1000 + dims + m)
    x = _data(rng, n, dims, **kw)
    q = _data(rng, 64, dims, **{k: v for k, v in kw.items() if k == "levels"})
    if metric == "cosine":
        x, q = x + 1.0, q + 1.0
    q[:8] = x[:8]
    labels = (rng.permutation(n).astype(np.uint64) << np.uint64(32)) | np.uint64(7)  # labels != ids
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    orc.build(x, labels)
    for i in range(0, n, 5):
        orc.mark_deleted(i)
    links, labs = orc.links(), orc.labels()
    ref = None
    if oracle_mod.available("ref"):
        ref = oracle_mod.FlatIndex("ref", dims, m, efc, 64, metric, capacity=n)
        ref.load_graph(x, links, labs)

    idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=n)
    idx.append(x, labs, links)
    assert idx.links().tobytes() == links.tobytes()
    for ef, coop in [(e, c) for e in efs for c in ("1", "0")]:
        with kernel_mode(coop):
            out = idx.search_batch(q, ef, want_stats=True)
        want = orc.search_many(q, ef, want_counters=True)
        assert out["n"].tolist() == want["n"].tolist(), (metric, ef, coop)
        assert out["labels"].tobytes() == want["labels"].tobytes(), (metric, ef, coop)
        if ref is not None:
            w2 = ref.search_many(q, ef, nthreads=2)
            assert out["labels"].tobytes() == w2["labels"].tobytes(), (metric, ef, "compiled reference")
        # identical traversal: same number of distance evals / expansions / link words as the oracle host saw
        assert out["stats"][:, 0].tolist() == want["counters"][:, 0].tolist()
        assert out["stats"][:, 1].tolist() == want["counters"][:, 1].tolist()
        assert out["stats"][:, 2].tolist() == want["counters"][:, 2].tolist()
        # distances of the returned nodes: bit-exact vs hnsw_dist_func on the same pairs
        for qi in range(0, q.shape[0], 7):
            k = int(out["n"][qi])
            ids = out["ids"][qi, :k]
            dd = oracle_mod.dist_many("port", metric, q[qi], x[ids]) if k else np.zeros(0, np.float32)
            assert out["dists"][qi, :k].tobytes() == dd.tobytes()
            assert (labs[ids] == out["labels"][qi, :k]).all()
    # the reference-shaped single-query entry point agrees with the batch
    one = idx.search(q[3], efs[-1])
    assert one.tolist() == orc.search(q[3], efs[-1]).tolist()
    idx.close()


def test_search_empty_and_tiny(pg, oracle_mod):
    idx = pg.HnswIndex(4, 3, 8, 8, "l2", capacity=8)
    out = idx.search_batch(np.zeros((3, 4), np.float32), 8)
    assert out["n"].tolist() == [0, 0, 0]                    # gh-2: empty index -> no rows
    assert idx.search(np.zeros(4, np.float32)).size == 0
    idx.insert(np.ones(4, np.float32), 42)
    assert idx.search(np.zeros(4, np.float32)).tolist() == [42]
    with pytest.raises(ValueError, match="Wrong number of dimensions"):   # embedding.c:311-315
        idx.search(np.zeros(5, np.float32))
    idx.close()


# ---------------------------------------------------------------------------------------------------
# a9-a11: bind (insert) -- link lists bit-for-bit
# ---------------------------------------------------------------------------------------------------
BIND_CFGS = [
    (3, 3, 16, 250, dict(levels=3)),
    (8, 4, 10, 500, dict(dup_frac=0.2)),
    (16, 8, 40, 1200, dict()),
    (33, 5, 20, 600, dict()),
    (128, 16, 64, 800, dict()),
    (24, 100, 16, 300, dict()),       # default m: lists never fill (append path only)
    (768, 4, 20, 300, dict()),
]


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("cfg", BIND_CFGS, ids=[f"d{c[0]}m{c[1]}n{c[3]}" for c in BIND_CFGS])
def test_bind_links_identical_to_oracle(pg, oracle_mod, metric, cfg):
    dims, m, efc, n, kw = cfg
    rng = np.random.default_rng(77 + dims * 3 + m)
    x = _data(rng, n, dims, **kw)
    if metric == "cosine":
        x = x + 1.0
    which = "ref" if oracle_mod.available("ref") else "port"
    orc = oracle_mod.FlatIndex(which, dims, m, efc, 64, metric, capacity=n)
    orc.build(x)
    idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=n)
    half = n // 2
    idx.insert_many(x[:half])                   # n sequential hnsw_add_point calls on the device
    for i in range(half, half + 5):
        idx.insert(x[i])                        # reference-shaped hnsw_bind_point, one at a time
    idx.insert_many(x[half + 5:])
    got, want = idx.links(), orc.links()
    bad = np.flatnonzero((got != want).any(1))
    assert bad.size == 0, f"{metric}: link lists differ at nodes {bad[:10]} (first: {got[bad[0]][:8]} vs {want[bad[0]][:8]})"
    # bulk build with batch_max=1 is the same sequence of exact binds (here with the throughput-mode kernel)
    idx2 = pg.HnswIndex(dims, m, efc, 64, metric, capacity=n)
    with kernel_mode("0"):
        idx2.build(x, batch_max=1)
    assert idx2.links().tobytes() == want.tobytes()
    idx.close()
    idx2.close()


# ---------------------------------------------------------------------------------------------------
# f1: reference record layout ingest / export
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims,m", [(3, 3), (33, 5), (128, 16)])
def test_record_layout_roundtrip(pg, oracle_mod, dims, m):
    rng = np.random.default_rng(5)
    n = 300
    x = _data(rng, n, dims)
    labels = rng.integers(0, 2**47, n).astype(np.uint64)
    orc = oracle_mod.FlatIndex("port", dims, m, 16, 64, "l2", capacity=n)
    orc.build(x, labels)
    recs = orc.records()
    idx = pg.HnswIndex(dims, m, 16, 64, "l2", capacity=n)
    idx.load_records(recs)
    assert idx.links().tobytes() == orc.links().tobytes()
    assert idx.labels().tobytes() == labels.tobytes()
    assert idx.export_records().tobytes() == recs.tobytes()
    q = _data(rng, 16, dims)
    assert idx.search_batch(q, 32)["labels"].tobytes() == orc.search_many(q, 32)["labels"].tobytes()
    idx.close()


# ---------------------------------------------------------------------------------------------------
# bulk build: structural validity + quality
# ---------------------------------------------------------------------------------------------------
def test_bulk_build_valid_graph_and_recall(pg, oracle_mod):
    rng = np.random.default_rng(9)
    n, dims, m, efc = 6000, 32, 8, 64
    x = _data(rng, n, dims)
    q = _data(rng, 200, dims)
    idx = pg.HnswIndex(dims, m, efc, 64, "l2", capacity=n)
    idx.build(x, batch_max=256)
    links = idx.links()
    cnt = links[:, 0]
    assert (cnt <= 2 * m).all() and (cnt[1:] > 0).all()
    for i in range(0, n, 37):
        l = links[i, 1:1 + cnt[i]]
        assert (l < n).all() and (l != i).all() and len(set(l.tolist())) == len(l)
    # the CPU reference algorithm searching the GPU-built graph returns exactly what the GPU returns
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, "l2", capacity=n)
    orc.load_graph(x, links)
    out = idx.search_batch(q, 64)
    assert out["labels"].tobytes() == orc.search_many(q, 64)["labels"].tobytes()
    # recall@10 vs exact brute force, compared with the reference's own sequential build
    d2 = ((q[:, None, :] - x[None, :, :]) ** 2).sum(-1)
    truth = np.argsort(d2, axis=1)[:, :10]
    def recall(labels):
        return np.mean([len(set(truth[i].tolist()) & set(labels[i, :10].tolist())) / 10 for i in range(len(q))])
    seq = oracle_mod.FlatIndex("port", dims, m, efc, 64, "l2", capacity=n)
    seq.build(x)
    r_gpu, r_seq = recall(out["labels"]), recall(seq.search_many(q, 64)["labels"])
    assert r_gpu > r_seq - 0.05, (r_gpu, r_seq)


# ---------------------------------------------------------------------------------------------------
# f2: scan iteration semantics (efSearch doubling, embedding.c:322-366)
# ---------------------------------------------------------------------------------------------------
SCAN_ITER_CFGS = [
    # dims, m, efC, n, data kwargs, efsearch, limit, deleted stride
    (8, 6, 24, 500, {}, 4, 60, 0),                       # doubling 4 -> 8 -> ... until the LIMIT is served
    (3, 3, 16, 300, {"levels": 3}, 2, None, 5),          # tie-heavy integer grid + deleted labels, scan to exhaustion
    (16, 4, 20, 700, {"dup_frac": 0.3}, 5, None, 0),     # duplicates; scan to exhaustion (n < efSearch ends it)
    (24, 5, 16, 64, {}, 64, None, 3),                    # first search already returns everything (n < efSearch)
]


@pytest.mark.parametrize("cfg", SCAN_ITER_CFGS, ids=[f"d{c[0]}n{c[3]}ef{c[5]}" for c in SCAN_ITER_CFGS])
def test_index_scan_iteration_equals_reference_loop(pg, oracle_mod, cfg):
    """hnsw_gettuple's loop (embedding.c:285-370) at the C ABI (pgemb_index_scan_*) against its restatement in oracle/scan_iter.c
    driving the checker's hnsw_search: same TIDs in the same order -- doubling, the count comparison of :338, qsort + bsearch
    de-duplication over a growing range (duplicates a probe misses are handed out twice by the reference, hence here too), deleted
    labels, the end-of-scan rule -- and the same number of searches.  TIDs use both 16-bit halves of the block number so that
    ItemPointerCompare's order differs from the numeric order of the label."""
    dims, m, efc, n, kw, efs, limit, del_stride = cfg
    rng = np.random.default_rng(1000 + dims + n)
    x = _data(rng, n, dims, **kw)
    # label = TID: block number spread over bi_hi / bi_lo, small offsets (several rows per page)
    blocks = rng.permutation(n * 3)[:n].astype(np.uint64) * np.uint64(977)
    labels = np.array([tid_label(int(b) & 0xffffffff, 1 + i % 7) for i, b in enumerate(blocks)], dtype=np.uint64)
    if del_stride:
        labels[::del_stride] |= np.uint64(1 << 48)
    for which in checkers(oracle_mod):
        orc = oracle_mod.FlatIndex(which, dims, m, efc, efs, "l2", capacity=n)
        orc.build(x, labels)
        idx = pg.HnswIndex(dims, m, efc, efs, "l2", capacity=n)
        idx.append(x, labels, orc.links())
        for qi in range(6):
            q = x[(qi * 37) % n] + np.float32(0.01 * qi)
            want = orc.scan(q, efs, limit)
            got = np.array(list(idx.scan(q, limit=limit)), dtype=np.uint64)
            assert got.tolist() == want["tids"].tolist(), (which, cfg, qi)
            assert idx.last_scan["searches"] == want["searches"] and idx.last_scan["ef"] == want["ef"]
            got_b = np.array(list(idx.scan(q, limit=limit, batch=7)), dtype=np.uint64)
            assert got_b.tolist() == got.tolist()
        assert idx.efsearch == efs                      # the doubled efSearch is the scan's own copy (embedding.c:254)
        idx.close()
        orc.close()


def check_ef_beyond_shared_memory(pg, oracle_mod, dims, n, efs):
    rng = np.random.default_rng(404)
    m, efc = 8, 40
    x = _data(rng, n, dims)
    q = _data(rng, 5, dims)
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, "cosine", capacity=n)
    orc.build(x + 1.0)
    idx = pg.HnswIndex(dims, m, efc, 64, "cosine", capacity=n)
    idx.append(x + 1.0, orc.labels(), orc.links())
    for ef in efs:
        out = idx.search_batch(q + 1.0, ef, want_stats=True)
        want = orc.search_many(q + 1.0, ef, want_counters=True)
        assert out["n"].tolist() == want["n"].tolist(), ef
        assert out["labels"].tobytes() == want["labels"].tobytes(), ef
        assert out["stats"][:, :3].tolist() == want["counters"][:, :3].tolist(), ef
    # and the scan that gets there by doubling: every node comes back exactly as the reference loop returns them
    want = orc.scan(q[0] + 1.0, 4096, None)
    got = list(idx.scan(q[0] + 1.0, efsearch=4096))
    assert got == want["tids"].tolist() and idx.last_scan["ef"] == want["ef"]
    idx.close()


def test_ef_beyond_shared_memory(pg, oracle_mod):
    """The reference doubles efSearch without bound (embedding.c:334): when 2 x ef keys no longer fit a CTA's shared memory
    (ef > ~12.6 K at 768-d) the traversal runs with its result queues in global memory -- same labels and counters as the oracle."""
    check_ef_beyond_shared_memory(pg, oracle_mod, 768, 3000, (20000, 13000, 64))


# ---------------------------------------------------------------------------------------------------
# K5: shard top-k merge
# ---------------------------------------------------------------------------------------------------
def test_merge_topk(pg):
    import ctypes as C
    import torch
    from pg_embedding_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(4)
    nq, S, k = 50, 4, 16
    d = np.sort(rng.integers(0, 20, size=(S, nq, k)).astype(np.float32), axis=2)  # many ties across shards
    l = rng.permutation(S * nq * k).astype(np.int64).reshape(S, nq, k)
    # within a shard list, equal distances must be in ascending label order (that is what search emits)
    for s in range(S):
        for qi in range(nq):
            order = np.lexsort((l[s, qi], d[s, qi]))
            d[s, qi], l[s, qi] = d[s, qi][order], l[s, qi][order]
    nin = rng.integers(0, k + 1, size=(S, nq)).astype(np.int32)
    td, tl, tn = torch.from_numpy(d).cuda(), torch.from_numpy(l).cuda(), torch.from_numpy(nin).cuda()
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    ol = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    on = torch.empty((nq,), dtype=torch.int32, device="cuda")
    st = lib.pgemb_merge_topk_device(nq, S, k, td.data_ptr(), tl.data_ptr(), tn.data_ptr(), od.data_ptr(), ol.data_ptr(),
                                     on.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert st == 0
    torch.cuda.synchronize()
    od, ol, on = od.cpu().numpy(), ol.cpu().numpy(), on.cpu().numpy()
    for qi in range(nq):
        pairs = sorted((float(d[s, qi, i]), int(l[s, qi, i])) for s in range(S) for i in range(nin[s, qi]))[:k]
        assert on[qi] == len(pairs)
        assert [(float(a), int(b)) for a, b in zip(od[qi, :on[qi]], ol[qi, :on[qi]])] == pairs


# ---------------------------------------------------------------------------------------------------
# BASELINE-sized checks: configs[1] against the oracle on a CPU-built graph, configs[2] (N=1M) through
# size-independent properties + an oracle sample on the GPU-built graph
# ---------------------------------------------------------------------------------------------------
def _clustered(rng, n, dim, centres):
    sigma = 0.3 * np.sqrt(2.0 * dim) / np.sqrt(dim)
    a = rng.integers(0, centres.shape[0], n)
    x = centres[a] + sigma * rng.standard_normal((n, dim)).astype(np.float32)
    return np.ascontiguousarray(x.astype(np.float32))


def test_config1_dims128_l2_vs_oracle(pg, oracle_mod):
    """BASELINE configs[1] at its full size (dims=128, N=100K, L2, m=16, efC=200, efS=64): the graph is built by the reference
    algorithm on the CPU (sequential, exact), searched by both; 4096 queries must match exactly (labels and traversal counters).
    The last 300 inserts are replayed on the GPU from the CPU's state before them: link lists bit-identical."""
    rng = np.random.default_rng(128)
    n, dims, m, efc, efs = 100_000, 128, 16, 200, 64
    centres = rng.standard_normal((316, dims)).astype(np.float32)
    x, q = _clustered(rng, n, dims, centres), _clustered(rng, 4096, dims, centres)
    which = "ref" if oracle_mod.available("ref") else "port"
    cut = n - 300
    orc = oracle_mod.FlatIndex(which, dims, m, efc, efs, "l2", capacity=n)
    orc.build(x[:cut])
    before = orc.records().copy()                        # the graph as it was before the last 300 inserts
    for i in range(cut, n):
        orc.add(x[i], i)
    idx = pg.HnswIndex(dims, m, efc, efs, "l2", capacity=n)
    idx.load_records(orc.records())
    out = idx.search_batch(q, efs, want_stats=True)
    want = orc.search_many(q, efs, nthreads=os.cpu_count() or 4, want_counters=True)
    assert out["labels"].tobytes() == want["labels"].tobytes()
    assert (out["stats"][:, :3].astype(np.uint64) == want["counters"]).all()
    idx2 = pg.HnswIndex(dims, m, efc, efs, "l2", capacity=n)
    idx2.load_records(before)
    idx2.insert_many(x[cut:])
    assert idx2.links().tobytes() == orc.links().tobytes()
    idx.close(); idx2.close()


def test_config2_full_size_properties(pg, oracle_mod):
    """BASELINE configs[2] at FULL size (dims=768, N=1M, cosine, m=32, efC=200, efS=64), GPU bulk build.
    Size-independent properties on 8192 queries + exact agreement with the CPU oracle on a 96-query sample."""
    torch = pytest.importorskip("torch")
    if torch.cuda.get_device_properties(0).total_memory < 40e9:
        pytest.skip("needs a large-memory GPU")
    import ctypes as C
    from pg_embedding_b200 import _lib
    lib = _lib.load()
    n, dims, m, efc, efs = 1_000_000, 768, 32, 200, 64
    g = torch.Generator(device="cuda"); g.manual_seed(7)
    centres = torch.randn((1000, dims), generator=g, device="cuda")
    def gen(k):
        a = torch.randint(0, 1000, (k,), generator=g, device="cuda")
        x = centres[a] + 0.424 * torch.randn((k, dims), generator=g, device="cuda")
        return x / x.norm(dim=1, keepdim=True)
    X = torch.cat([gen(250_000) for _ in range(4)])
    Q = gen(8192)
    idx = pg.HnswIndex(dims, m, efc, efs, "cosine", capacity=n)
    _lib.check(lib.pgemb_index_append_device(idx.dev, n, X.data_ptr(), None, None, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    idx.build_appended(0, n, 4096)
    q = Q.cpu().numpy()
    out = idx.search_batch(q, efs, want_stats=True)
    again = idx.search_batch(q, efs)
    assert out["labels"].tobytes() == again["labels"].tobytes()            # idempotent / deterministic
    assert (out["n"] == efs).all()
    d, ids = out["dists"], out["ids"]
    assert (np.diff(d, axis=1) >= 0).all()                                 # ascending by distance
    assert all(len(set(r.tolist())) == efs for r in ids[::64])             # distinct nodes
    assert (out["labels"] == ids).all()                                    # label == id here
    re = idx.dist_gather(q[:512], ids[:512])                               # distances recomputed pair by pair
    assert re.tobytes() == d[:512].tobytes()
    assert (out["stats"][:, 0] >= efs).all() and (out["stats"][:, 1] >= 1).all()
    # graph structure
    links = idx.links(0, 200_000)
    assert (links[:, 0] <= 2 * m).all() and (links[1:, 0] > 0).all()
    # oracle sample on the identical graph (reference record layout exported from HBM)
    which = "ref" if oracle_mod.available("ref") else "port"
    orc = oracle_mod.FlatIndex(which, dims, m, efc, efs, "cosine", capacity=n)
    for s in range(0, n, 1 << 16):
        orc.load_records(idx.export_records(s, min(1 << 16, n - s)))
    want = orc.search_many(q[:96], efs, nthreads=min(96, os.cpu_count() or 4), want_counters=True)
    assert out["labels"][:96].tobytes() == want["labels"].tobytes()
    assert (out["stats"][:96, :3].astype(np.uint64) == want["counters"]).all()
    idx.close()


# ---------------------------------------------------------------------------------------------------
# exact parallel build: speculative batches must reproduce the sequential reference build bit for bit
# ---------------------------------------------------------------------------------------------------
EXACT_CFGS = [
    (3, 3, 16, 400, dict(levels=3), "l2"),            # ties + duplicates: conflicts everywhere
    (16, 8, 40, 3000, dict(), "cosine"),
    (32, 8, 64, 6000, dict(), "l2"),
    (128, 16, 100, 4000, dict(), "manhattan"),
    (768, 32, 200, 1500, dict(), "cosine"),
    (5, 0, 8, 300, dict(), "manhattan"),              # m=0: no back-links, so nothing to validate
]


@pytest.mark.parametrize("cfg", EXACT_CFGS, ids=[f"d{c[0]}m{c[1]}n{c[3]}{c[5]}" for c in EXACT_CFGS])
def test_exact_parallel_build_equals_sequential(pg, oracle_mod, cfg):
    dims, m, efc, n, kw, metric = cfg
    rng = np.random.default_rng(4242 + dims)
    x = _data(rng, n, dims, **kw)
    if metric == "cosine":
        x = x + 1.0
    which = "ref" if oracle_mod.available("ref") else "port"
    orc = oracle_mod.FlatIndex(which, dims, m, efc, 64, metric, capacity=n)
    orc.build(x)
    want = orc.links()
    for bmax in (64, 1024):
        idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=n)
        idx.append(x)
        secs, st = idx.build_exact(0, n, bmax)
        got = idx.links()
        bad = np.flatnonzero((got != want).any(1))
        assert bad.size == 0, f"{metric} bmax={bmax}: link lists differ at nodes {bad[:10]}; stats {st}"
        assert st["searches"] >= n - 1 and st["batches"] <= n
        idx.close()


# ---------------------------------------------------------------------------------------------------
# edge parameters: dims=1, m=0/1, ef far above N and above 1000 (queue buffers scale), odd dims
# ---------------------------------------------------------------------------------------------------
EDGE_CFGS = [
    (1, 1, 4, 200, "l2", (1, 7, 1000)),
    (5, 0, 8, 50, "manhattan", (1, 64)),            # m=0: maxM=0, no links at all (reloption minimum, embedding.c:132)
    (7, 2, 300, 500, "cosine", (3, 600)),           # efconstruction > N for most of the build
    (2000, 2, 8, 60, "l2", (16,)),                  # largest dims a page can hold (embedding.c:229-231)
    (1999, 3, 8, 60, "cosine", (16,)),
]


@pytest.mark.parametrize("cfg", EDGE_CFGS, ids=[f"d{c[0]}m{c[1]}n{c[3]}{c[4]}" for c in EDGE_CFGS])
def test_edge_parameters(pg, oracle_mod, cfg):
    dims, m, efc, n, metric, efs = cfg
    rng = np.random.default_rng(dims * 31 + m)
    x = rng.standard_normal((n, dims)).astype(np.float32) + (1.5 if metric == "cosine" else 0.0)
    q = rng.standard_normal((16, dims)).astype(np.float32) + (1.5 if metric == "cosine" else 0.0)
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    orc.build(x)
    idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=n)
    idx.insert_many(x)
    assert idx.links().tobytes() == orc.links().tobytes()
    for ef in efs:
        out = idx.search_batch(q, ef)
        want = orc.search_many(q, ef)
        assert out["n"].tolist() == want["n"].tolist()
        assert out["labels"].tobytes() == want["labels"].tobytes()
    idx.close()


# ---------------------------------------------------------------------------------------------------
# f3: exact scan (what ORDER BY val <op> q LIMIT k returns without the index; knn.out:63-91)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_scan_topk_matches_exact_order(pg, oracle_mod, metric):
    rng = np.random.default_rng(99)
    for dims, n, k, levels in ((3, 500, 7, 3), (33, 3000, 64, 0), (128, 20000, 10, 0), (203, 4000, 10, 0), (768, 1500, 10, 0)):
        x = _data(rng, n, dims, levels=levels)
        q = _data(rng, 24, dims, levels=levels)
        if metric == "cosine":
            x, q = x + 1.0, q + 1.0
        labels = rng.permutation(n).astype(np.uint64) + np.uint64(5)
        idx = pg.HnswIndex(dims, 4, 8, 16, metric, capacity=n)
        idx.append(x, labels)
        dead = np.arange(0, n, 9)
        idx.mark_deleted(dead)
        out = idx.scan_topk(q, k)
        alive = np.ones(n, bool); alive[dead] = False
        for i in range(q.shape[0]):
            d = oracle_mod.dist_many("port", metric, q[i], x)
            order = sorted((float(d[j]), int(labels[j])) for j in range(n) if alive[j])[:k]
            c = int(out["n"][i])
            assert c == len(order)
            assert out["labels"][i, :c].tolist() == [o[1] for o in order], (metric, dims, i)
            assert out["dists"][i, :c].tobytes() == np.array([o[0] for o in order], np.float32).tobytes()
        idx.close()


def test_scan_topk_regress_seqscan(pg):
    """knn.out:63-91: the seq-scan orders of the regress table for the three operators."""
    case = GOLD[0]
    for metric, want in case["expected"].items():
        idx = pg.HnswIndex(3, 3, 16, 64, metric, capacity=8)
        rows = case["rows"]
        idx.append(np.array([r["val"] for r in rows], np.float32), np.array([tid_label(*r["tid"]) for r in rows], np.uint64))
        out = idx.scan_topk(np.array([case["query"]], np.float32), 4)
        by_label = {tid_label(*r["tid"]): r["val"] for r in rows}
        assert [by_label[int(l)] for l in out["labels"][0, : out["n"][0]]] == want, metric
        idx.close()


# ---------------------------------------------------------------------------------------------------
# growth: a relation grows page by page (embedding.c:636-691), the device index with it
# ---------------------------------------------------------------------------------------------------
def check_reserve_keeps_contents_and_ids(pg, oracle_mod):
    """Body shared by tests/test_capi_emulated.py (emulated library) and the GPU test at the end of tests/test_sidecar.py."""
    rng = np.random.default_rng(31)
    n, dims, m, efc = 260, 12, 4, 16
    for metric in ("cosine", "l2"):
        x = rng.standard_normal((n, dims)).astype(np.float32) + (1.0 if metric == "cosine" else 0.0)
        orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
        orc.build(x)
        idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=40)
        idx.insert_many(x[:40])                                  # full
        with pytest.raises(Exception):
            idx.insert_many(x[40:41])
        idx.reserve(30)                                          # smaller: no-op
        idx.reserve(150)
        q = rng.standard_normal((9, dims)).astype(np.float32) + (1.0 if metric == "cosine" else 0.0)
        idx.insert_many(x[40:150])                               # binds see the old nodes at their old ids
        idx.reserve(n)
        idx.insert_many(x[150:])
        assert idx.links().tobytes() == orc.links().tobytes(), metric
        assert idx.labels().tobytes() == orc.labels().tobytes()
        for coop in ("1", "0"):                                  # visited bitmaps were re-made for the new capacity
            with kernel_mode(coop):
                out = idx.search_batch(q, 500)                   # ef > 4096-entry hash's half -> exercises the bitmap too on small tables
            assert out["labels"].tobytes() == orc.search_many(q, 500)["labels"].tobytes(), (metric, coop)
        idx.close()

