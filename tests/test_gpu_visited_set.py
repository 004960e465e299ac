"""GPU tests of the traversal's per-slot visited set (search_kernel.cuh, K3) in each of its regimes, against the C oracle.

Whether a neighbour is scored depends on the visited set, a small state machine per slot:
a. a global open-addressing table updated by atomicCAS at L2 -- used only when the capacity's bitmap is larger than the table
   (capi.cu visited_hash_entries), so never at the capacities the parity tests use;
b. in latency mode, a table in the CTA's shared memory instead (PGEMB_SMEM_VISITED);
c. the migration of either table to the exact N-bit bitmap before it passes half full (__ldcg of the table, plain stores to
   clear it, bitmap bits set, the log rewritten from table positions to ids);
d. the reset after each query from the slot's log, or a full clear of the bitmap when a traversal visited more than the log
   holds (`vlog_cap`, capi.cu ensure_workspace);
e. slot reuse: a throughput-mode slot serves one query after another, and the workspace survives across calls, so every
   reset is what the slot's next query starts from.

A stale visited bit or table entry crashes nothing: the next query on that slot skips a node and returns other neighbours
or takes another path.  So every case asserts what `test_search_identical_to_oracle` asserts (n and labels byte-identical,
the traversal counters stats[:, :3] equal to the oracle's, the distances of the returned nodes bit-identical to
hnsw_dist_func), and then asserts that it reached the regime it claims, from stats[:, 0]: the kernel adds a hop's admitted
nodes to stats[:, 0] and to the slot's log alike (`st_dist += n`, `logn += popc`), so stats[:, 0] is the number of nodes the
visited set admitted -- the entry point plus every unvisited neighbour -- and that is the length of the slot's log.

The graphs are built by the oracle and loaded into a device index whose capacity selects the mode.  tests/test_capi_emulated.py
runs the migration, reset, tie and layout-sequence bodies on the host-emulated library at small sizes; the log-overflow
cases need more than 32 768 visits per query and stay on the GPU, where the emulator would take too long."""
import functools
import os

import numpy as np
import pytest

from test_gpu_parity import METRICS, _data

pytestmark = pytest.mark.gpu

VLOG_MAX = 32768             # ensure_workspace: the log holds min(capacity, 32768) ids, at least half a table
KNOBS = ("COOP", "SMEM_VISITED", "VISITED_HASH", "VH_PER_EF", "VISITED_PAIRS", "WARPS", "RES_GLOBAL")


@pytest.fixture(scope="module")
def pg():
    import pg_embedding_b200 as pg
    from pg_embedding_b200 import build
    build.build()
    if pg.device_count() < 1:
        pytest.fail("no CUDA device: the product path has no CPU fallback")
    return pg


@pytest.fixture(scope="module")
def sms(pg):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- the sizing rules, mirrored --------------------------------------------------------------------------------------
def hash_entries(capacity, ef, vh_per_ef=64, hash_on=True):
    """visited_hash_entries() in csrc/capi.cu: entries H of a slot's global table, 0 when the bitmap is the smaller structure."""
    want = max(ef * vh_per_ef, 4096)
    h = 4096
    while h < want and h < (1 << 20):
        h <<= 1
    bitmap_bytes = (capacity + 31) // 32 * 4
    return h if hash_on and bitmap_bytes > 4 * h else 0


def vlog_cap(capacity, vh_max, vhs=0):
    """ensure_workspace() in csrc/capi.cu: the capacity of a slot's log.  The workspace only grows, so vh_max is the largest
    table this index's workspace was sized for (and vhs the shared-memory table of the call); the result is an upper bound."""
    return max(min(capacity, VLOG_MAX), vh_max // 2, vhs // 2)


def set_knobs(monkeypatch, **kv):
    """Every visited-set switch of launch_search set for this call: the given PGEMB_<name> values, the rest at their defaults."""
    for k in KNOBS:
        v = kv.get(k)
        if v is None:
            monkeypatch.delenv("PGEMB_" + k, raising=False)
        else:
            monkeypatch.setenv("PGEMB_" + k, str(v))


def assert_migrates(visits, H, maxm, frac, mixed=False, what=""):
    """Visits above H/2 + maxM: the table passed the migration test (logn + cnt > H/2) on some hop.  Below H/2 - maxM: it never
    did.  `frac` of the queries (at least one) must be of each kind claimed."""
    assert H > 0, what
    need = max(1, int(frac * len(visits)))
    above, below = int((visits > H // 2 + maxm).sum()), int((visits < H // 2 - maxm).sum())
    assert above >= need, (what, "migrated", above, "of", len(visits), "H", H, np.percentile(visits, [0, 50, 100]))
    if mixed:
        assert below >= need, (what, "unmigrated", below, "of", len(visits), "H", H, np.percentile(visits, [0, 50, 100]))


# ---- graphs and the oracle comparison --------------------------------------------------------------------------------
class Graph:
    pass


@functools.lru_cache(maxsize=None)
def graph(oracle_mod, metric, dims, m, efc, n, nq, levels=0, dup_frac=0.0, seed=0):
    """An oracle-built graph with labels != ids, its oracle(s), and nq queries."""
    rng = np.random.default_rng(seed + 1000 * dims + n)
    x = _data(rng, n, dims, levels=levels, dup_frac=dup_frac)
    q = _data(rng, nq, dims, levels=levels)
    if metric == "cosine":
        x, q = x + 1.0, q + 1.0
    q[:4] = x[:4]
    g = Graph()
    g.metric, g.dims, g.m, g.efc, g.maxm, g.x, g.q = metric, dims, m, efc, 2 * m, x, q
    g.labels = (rng.permutation(n).astype(np.uint64) << np.uint64(32)) | np.uint64(3)
    g.orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    g.orc.build(x, g.labels)
    g.links = g.orc.links()
    g.ref = None
    if oracle_mod.available("ref"):
        g.ref = oracle_mod.FlatIndex("ref", dims, m, efc, 64, metric, capacity=n)
        g.ref.load_graph(x, g.links, g.labels)
    return g


def load(pg, g, capacity):
    idx = pg.HnswIndex(g.dims, g.m, g.efc, 64, g.metric, capacity=capacity)
    idx.append(g.x, g.labels, g.links)
    return idx


def check(idx, oracle_mod, g, q, ef, what):
    """One search_batch against the oracle at the bar of test_search_identical_to_oracle; returns stats[:, 0] (visits)."""
    out = idx.search_batch(q, ef, want_stats=True)
    want = g.orc.search_many(q, ef, nthreads=os.cpu_count() or 4, want_counters=True)
    assert out["n"].tolist() == want["n"].tolist(), what
    bad = np.flatnonzero((out["labels"] != want["labels"]).any(1))
    assert bad.size == 0, (what, "labels differ for queries", bad[:8])
    if g.ref is not None:
        w2 = g.ref.search_many(q, ef, nthreads=os.cpu_count() or 4)
        assert out["labels"].tobytes() == w2["labels"].tobytes(), (what, "compiled reference")
    bad = np.flatnonzero((out["stats"][:, :3].astype(np.uint64) != want["counters"]).any(1))
    assert bad.size == 0, (what, "traversal counters differ for queries", bad[:8], out["stats"][bad[:2], :3], want["counters"][bad[:2]])
    for qi in range(q.shape[0]):
        k = int(out["n"][qi])
        ids = out["ids"][qi, :k]
        dd = oracle_mod.dist_many("port", g.metric, q[qi], g.x[ids]) if k else np.zeros(0, np.float32)
        assert out["dists"][qi, :k].tobytes() == dd.tobytes(), (what, qi)
        assert (g.labels[ids] == out["labels"][qi, :k]).all(), (what, qi)
    return out["stats"][:, 0].astype(np.int64), out


def reuse_batch(g, slots):
    """At least three queries per slot (the graph's queries repeated if needed): every slot serves several in one launch."""
    nq = 3 * slots + 5
    reps = -(-nq // g.q.shape[0])
    return np.ascontiguousarray(np.tile(g.q, (reps, 1))[:nq])


# ---- bodies (sizes are parameters: tests/test_capi_emulated.py calls them small) -------------------------------------
# ef at which a third to a half of the queries pass 2 048 visits, by n (16-d, m 8).  The GPU runs n 40 000: ~2 000 visits there
# leave most 32-id bitmap words with a single visited id, so a reset that skips one id leaves a bit that its word's other ids
# do not clear by accident
MIG_EF = {4000: {"l2": 1200, "cosine": 1200, "manhattan": 1000}, 40000: {"l2": 800, "cosine": 850, "manhattan": 750}}


def check_migration_throughput(pg, oracle_mod, metric, monkeypatch, sms, warps=1, n=40000, frac=0.1):
    """Throughput mode (search_kernel<M, COOP=false>), global table of H = 4096 entries (PGEMB_VH_PER_EF=1), nq >= 3 x slots:
    each slot alternates between queries that migrate at L2 and queries that do not.  Then the same batch on the bitmap alone
    (PGEMB_VISITED_HASH=0): same counters."""
    g = graph(oracle_mod, metric, 16, 8, 40, n, 64)
    cap, ef = 1 << 18, MIG_EF[n][metric]
    slots = warps * sms
    q = reuse_batch(g, slots)
    assert q.shape[0] >= 3 * slots
    idx = load(pg, g, cap)
    set_knobs(monkeypatch, COOP=0, WARPS=warps, VH_PER_EF=1)
    H = hash_entries(cap, ef, vh_per_ef=1)
    assert H == 4096
    v, _ = check(idx, oracle_mod, g, q, ef, "hash, migration mid-batch")
    assert_migrates(v, H, g.maxm, frac, mixed=True, what=metric)
    set_knobs(monkeypatch, COOP=0, WARPS=warps, VISITED_HASH=0)
    assert hash_entries(cap, ef, hash_on=False) == 0
    v2, _ = check(idx, oracle_mod, g, q, ef, "bitmap only")
    assert (v2 == v).all()
    idx.close()


def check_latency_global_hash(pg, oracle_mod, metric, monkeypatch, sms, pairs, n=40000, nq=64, frac=0.1):
    """Latency mode (search_kernel<M, COOP=true>) with the table at L2 (PGEMB_SMEM_VISITED=0, H = 4096): the paired
    (PGEMB_VISITED_PAIRS=1, two atomicCAS probes in flight) or ordered test-and-set, and their migration.  Launches of at most
    one query per SM; the CTAs of later launches start from the resets of earlier ones."""
    g = graph(oracle_mod, metric, 16, 8, 40, n, 64)
    cap, ef = 1 << 18, MIG_EF[n][metric]
    idx = load(pg, g, cap)
    set_knobs(monkeypatch, SMEM_VISITED=0, VH_PER_EF=1, VISITED_PAIRS=pairs)
    per = min(sms, nq)
    vs = []
    for lo in range(0, nq, per):
        qq = g.q[np.arange(lo, lo + per) % g.q.shape[0]]
        vs.append(check(idx, oracle_mod, g, qq, ef, ("latency, global hash", pairs, lo))[0])
    assert_migrates(np.concatenate(vs), hash_entries(cap, ef, vh_per_ef=1), g.maxm, frac, mixed=True, what=(metric, pairs))
    idx.close()


def check_latency_small_smem_table(pg, oracle_mod, metric, monkeypatch, sms, n=4000, nq=64, ef=300, frac=0.5):
    """Latency mode with a 1024-entry table in shared memory (PGEMB_SMEM_VISITED=1024): it migrates after 512 visits."""
    g = graph(oracle_mod, metric, 16, 8, 40, n, 64)
    idx = load(pg, g, 1 << 18)
    set_knobs(monkeypatch, SMEM_VISITED=1024)
    per = min(sms, nq)
    vs = []
    for lo in range(0, nq, per):
        qq = g.q[np.arange(lo, lo + per) % g.q.shape[0]]
        vs.append(check(idx, oracle_mod, g, qq, ef, ("latency, shared-memory table", lo))[0])
    assert_migrates(np.concatenate(vs), 1024, g.maxm, frac, what=metric)
    idx.close()


def check_ties(pg, oracle_mod, metric, monkeypatch, sms, n=2000, warps=1):
    """Integer grid with duplicates (3-d, 3 levels) on a hash-mode capacity, throughput mode with slot reuse: the tie overflow
    buffer (stats[:, 3], its high-water mark) and the visited reset of the same slot, query after query."""
    g = graph(oracle_mod, metric, 3, 3, 16, n, 64, levels=3, dup_frac=0.2)
    cap = 1 << 21
    idx = load(pg, g, cap)
    set_knobs(monkeypatch, COOP=0, WARPS=warps)
    q = reuse_batch(g, warps * sms)
    for ef in (16, 64):
        H = hash_entries(cap, ef)
        assert H >= 4096
        v, out = check(idx, oracle_mod, g, q, ef, ("ties", ef))
        assert (v < H // 2 - g.maxm).all()
        assert (out["stats"][:, 3] > 0).any(), ("no query overflowed the tie buffer", ef)
    idx.close()


def check_layout_sequence(pg, oracle_mod, metric, monkeypatch, sms, dims, m, efc, n, ef_mig, ef_overflow=None, nq=64, frac=0.1):
    """One index, one call after another, each against the oracle, each with a different visited-set layout: log overflow
    (full clear), then small ef in throughput mode on the same slots; the table stride 1 x ef <-> 64 x ef inside an allocation
    made for the larger table; PGEMB_WARPS 1 <-> default; latency <-> throughput mode; table <-> bitmap only.  No call may leave
    state behind that a later call with another layout trips over."""
    g = graph(oracle_mod, metric, dims, m, efc, n, 64)
    cap = 1 << 21
    idx = load(pg, g, cap)
    some_q = g.q[:nq]
    small_q = g.q[: min(sms, g.q.shape[0])]
    reuse_q = reuse_batch(g, sms)
    vh_max = 0
    steps = []
    if ef_overflow:
        steps += [(dict(VH_PER_EF=1), ef_overflow, some_q, "overflow")]
    steps += [
        (dict(COOP=0, WARPS=1), 64, reuse_q, "none"),
        (dict(COOP=0, WARPS=1, VISITED_HASH=0), 64, reuse_q, "none"),
        (dict(COOP=0, WARPS=1, VH_PER_EF=1), ef_mig, reuse_q, "migrate"),
        (dict(COOP=0), 256, some_q, "none"),
        (dict(COOP=1, SMEM_VISITED=0), 256, small_q, "none"),
        (dict(COOP=1, SMEM_VISITED=0, VH_PER_EF=1), ef_mig, small_q, "migrate"),
        (dict(COOP=0, WARPS=1, VISITED_HASH=0), ef_mig, reuse_q, "none"),
    ]
    if ef_overflow:
        steps += [(dict(VISITED_HASH=0), ef_overflow, some_q, "overflow")]
    steps += [(dict(COOP=0, WARPS=1), 64, reuse_q, "none"), (dict(COOP=1), 64, small_q, "none")]
    for i, (knobs, ef, q, claim) in enumerate(steps):
        set_knobs(monkeypatch, **knobs)
        H = hash_entries(cap, ef, vh_per_ef=knobs.get("VH_PER_EF", 64), hash_on=knobs.get("VISITED_HASH", 1) != 0)
        vh_max = max(vh_max, H)
        v, _ = check(idx, oracle_mod, g, q, ef, (i, knobs, ef))
        if claim == "migrate":
            assert_migrates(v, H, g.maxm, frac, what=(i, knobs))
        elif claim == "overflow":
            assert (v > vlog_cap(cap, vh_max)).mean() >= 0.25, (i, knobs, vlog_cap(cap, vh_max), np.percentile(v, [0, 50, 100]))
    idx.close()


# ---- search cases ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", METRICS)
def test_throughput_global_hash_no_migration(pg, oracle_mod, sms, metric, monkeypatch):
    """The production mode at small ef: capacity 2^21, default PGEMB_VH_PER_EF, ef 64 and 256 (tables of 4096 and 16384)."""
    g = graph(oracle_mod, metric, 16, 8, 40, 4000, 64)
    cap = 1 << 21
    idx = load(pg, g, cap)
    set_knobs(monkeypatch, COOP=0)
    q = reuse_batch(g, sms)
    for ef in (64, 256):
        H = hash_entries(cap, ef)
        assert H == 64 * ef
        v, _ = check(idx, oracle_mod, g, q, ef, ef)
        assert (v < H // 2 - g.maxm).all()
    idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("warps", [1, 2])
def test_throughput_migration_with_slot_reuse(pg, oracle_mod, sms, metric, warps, monkeypatch):
    check_migration_throughput(pg, oracle_mod, metric, monkeypatch, sms, warps=warps)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("pairs", [0, 1])
def test_latency_global_hash(pg, oracle_mod, sms, metric, pairs, monkeypatch):
    check_latency_global_hash(pg, oracle_mod, metric, monkeypatch, sms, pairs)


@pytest.mark.parametrize("metric", METRICS)
def test_latency_small_shared_memory_table(pg, oracle_mod, sms, metric, monkeypatch):
    check_latency_small_smem_table(pg, oracle_mod, metric, monkeypatch, sms)


LOG_EF = 30000      # 8-d, n 60 000, m 4: 32 000 - 41 000 visits, past the 32 768-id log


@pytest.mark.parametrize("metric", METRICS)
def test_log_overflow_full_clear(pg, oracle_mod, metric, monkeypatch):
    """search_kernel<M, false, 4, RESG=true> (result queues in global memory): the table (H = 32768 with PGEMB_VH_PER_EF=1)
    migrates, the traversal passes vlog_cap, and the reset is the full clear.  Then the same graph in a bitmap-only index
    (capacity 131 072): the full clear without a table.  Two calls of 32 queries each with one warp per CTA: both run on slots
    0-31, so every query of the second call starts from a full clear of the first."""
    g = graph(oracle_mod, metric, 8, 4, 16, 60000, 64)
    for cap, knobs in ((1 << 21, dict(RES_GLOBAL=1, VH_PER_EF=1, WARPS=1)), (1 << 17, dict(WARPS=1))):
        set_knobs(monkeypatch, **knobs)
        idx = load(pg, g, cap)
        H = hash_entries(cap, LOG_EF, vh_per_ef=knobs.get("VH_PER_EF", 64))
        assert H == (32768 if cap == 1 << 21 else 0)
        for half in (g.q[:32], g.q[32:]):
            v, _ = check(idx, oracle_mod, g, half, LOG_EF, (cap, knobs))
            if H:
                assert_migrates(v, H, g.maxm, 1.0, what=cap)
            assert (v > vlog_cap(cap, H)).mean() >= 0.25, (cap, np.percentile(v, [0, 50, 100]))
        idx.close()


@pytest.mark.parametrize("coop", [0, 1])
def test_l2_eight_lanes_with_hash(pg, oracle_mod, sms, coop, monkeypatch):
    """search_kernel<M_L2, COOP, TPR=8> (1536-d rows) on a global table of 4096 entries that every query migrates.  ef 1500:
    at ef 1024 these queries visit 1 550 - 1 900 nodes, short of the 2 048 that migration needs."""
    g = graph(oracle_mod, "l2", 1536, 8, 32, 3000, 64)
    cap, ef = 1 << 18, 1500
    idx = load(pg, g, cap)
    set_knobs(monkeypatch, COOP=coop, VH_PER_EF=1, SMEM_VISITED=0)
    q = g.q if coop == 0 else g.q[: min(sms, 64)]
    v, _ = check(idx, oracle_mod, g, q, ef, ("tpr8", coop))
    assert_migrates(v, hash_entries(cap, ef, vh_per_ef=1), g.maxm, 0.5)
    idx.close()


@pytest.mark.parametrize("metric", METRICS)
def test_ties_with_slot_reuse(pg, oracle_mod, sms, metric, monkeypatch):
    check_ties(pg, oracle_mod, metric, monkeypatch, sms)


@pytest.mark.parametrize("metric", METRICS)
def test_one_index_changing_layouts(pg, oracle_mod, sms, metric, monkeypatch):
    check_layout_sequence(pg, oracle_mod, metric, monkeypatch, sms, 8, 4, 16, 60000, ef_mig=1200, ef_overflow=LOG_EF)


# ---- insert and build cases ------------------------------------------------------------------------------------------
BIND = (32, 16, 300, 3000)      # dims, m, efC, n: uniform 32-d data, bind searches at ef 300 visit 2 100 - 2 300 nodes


def bind_graph(oracle_mod, metric):
    dims, m, efc, n = BIND
    rng = np.random.default_rng(5 + dims)
    x = rng.standard_normal((n, dims)).astype(np.float32) + (1.0 if metric == "cosine" else 0.0)
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    orc.build(x)
    # a bind's search is not reported; the oracle's search of the finished graph at ef = efC from the inserted rows stands in
    v = orc.search_many(x[::10], efc, nthreads=os.cpu_count() or 4, want_counters=True)["counters"][:, 0].astype(np.int64)
    return x, orc, v


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("knobs", [dict(), dict(SMEM_VISITED=0), dict(COOP=0)], ids=["latency", "latency-l2-table", "throughput"])
def test_insert_on_hash_index(pg, oracle_mod, metric, knobs, monkeypatch):
    """insert_many (pgemb_insert_batch) and insert (hnsw_bind_point) into a hash-mode index (capacity 2^18, H = 4096): link
    lists byte for byte equal to the oracle's sequential build."""
    dims, m, efc, n = BIND
    x, orc, v = bind_graph(oracle_mod, metric)
    cap = 1 << 18
    set_knobs(monkeypatch, VH_PER_EF=1, **knobs)
    assert_migrates(v, hash_entries(cap, efc, vh_per_ef=1), 2 * m, 0.5)
    idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=cap)
    half = n // 2
    idx.insert_many(x[:half])
    for i in range(half, half + 5):
        idx.insert(x[i])
    idx.insert_many(x[half + 5:])
    got, want = idx.links(), orc.links()
    bad = np.flatnonzero((got != want).any(1))
    assert bad.size == 0, (metric, knobs, "link lists differ at nodes", bad[:10])
    idx.close()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("cap,vh_per_ef", [(1 << 21, None), (1 << 18, 1)], ids=["2^21", "2^18-migrating"])
def test_build_exact_on_hash_index(pg, oracle_mod, metric, cap, vh_per_ef, monkeypatch):
    """pgemb_build_exact with batches of up to 1024 searches (throughput mode) on the global table: the sequential graph."""
    dims, m, efc, n = BIND
    x, orc, v = bind_graph(oracle_mod, metric)
    set_knobs(monkeypatch, VH_PER_EF=vh_per_ef)
    H = hash_entries(cap, efc, vh_per_ef=vh_per_ef or 64)
    assert H > 0
    if vh_per_ef == 1:
        assert_migrates(v, H, 2 * m, 0.5)
    idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=cap)
    idx.append(x)
    _, st = idx.build_exact(0, n, 1024)
    bad = np.flatnonzero((idx.links() != orc.links()).any(1))
    assert bad.size == 0, (metric, cap, "link lists differ at nodes", bad[:10], st)
    idx.close()


@pytest.mark.parametrize("metric", METRICS)
def test_reserve_across_the_hash_threshold(pg, oracle_mod, metric, monkeypatch):
    """Capacity 100 000 (bitmap only), inserts, reserve(300 000) (a 4096-entry table from then on), more inserts: the links and
    a migrating search equal the oracle's."""
    dims, m, efc, n = BIND
    x, orc, v = bind_graph(oracle_mod, metric)
    set_knobs(monkeypatch, VH_PER_EF=1)
    assert hash_entries(100_000, efc, vh_per_ef=1) == 0 and hash_entries(300_000, efc, vh_per_ef=1) == 4096
    idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=100_000)
    idx.insert_many(x[: n // 2])
    idx.reserve(300_000)
    idx.insert_many(x[n // 2:])
    bad = np.flatnonzero((idx.links() != orc.links()).any(1))
    assert bad.size == 0, (metric, "link lists differ at nodes", bad[:10])
    g = Graph()
    g.metric, g.x, g.labels, g.orc, g.ref, g.maxm = metric, x, orc.labels(), orc, None, 2 * m
    q = x[1::23][:64] + np.float32(0.01)
    vv, _ = check(idx, oracle_mod, g, q, efc, "after reserve")
    assert_migrates(vv, 4096, 2 * m, 0.5)
    idx.close()
