"""GPU tests of the bulk build (`pgemb_build_bulk`, capi.cu) against the oracle's model of it, byte for byte.

The bulk build binds nodes in batches: every member of a batch runs bindPoint's search against the graph as it was when the
batch started, then writes its own list, and back-links are applied per target in source-id order.  Batch members are
unreachable in that snapshot (blank lists, named by no list), so the batch is exactly "search every member, then
mutuallyConnectNewElement for each member in id order" -- `oracle_bind_batch` in oracle/hnsw_oracle.c, driven through the
build's batch schedule by `FlatIndex.build_bulk`.  Every case here asserts:
- the device's link lists equal the model's byte for byte, for every node;
- the batch schedule reaches the sizes the case claims (the kernel paths depend on the batch size: one node sorts nothing,
  up to 8 run the staged select, larger batches the unstaged select and the cub sort of their (target, source) pairs);
- a search of the built graph equals the oracle's search of the same graph: labels, the traversal counters stats[:, :3] and
  the distance bits (`check` of tests/test_gpu_visited_set.py).

A valid graph with the sequential build's recall is not enough: back-links applied in the wrong source order, a full list
re-pruned against a stale copy, a drifted schedule or a search that sees a batch-mate all give one.  tests/test_oracle_bulk_model.py
shows on the same data that the model differs from the sequential build whenever batch_max > 1, so the comparison is not
vacuous.  tests/test_capi_emulated.py runs the bodies on the host-emulated library at n <= 500."""
import contextlib

import numpy as np
import pytest

from test_gpu_parity import _data, kernel_mode
from test_gpu_visited_set import Graph, check

pytestmark = pytest.mark.gpu

BATCH_MAX = [1, 8, 64, 4096]

CASES = [
    # id, metric, dims, m, efC, n, data kwargs.  n >= 2200: batch_max 64 is reached and 4096 gives batches above 64
    ("l2-d16", "l2", 16, 8, 40, 3000, dict()),
    ("cosine-d16", "cosine", 16, 8, 40, 3000, dict()),
    ("manhattan-d16", "manhattan", 16, 8, 40, 3000, dict()),
    ("ties-l2", "l2", 3, 3, 16, 2500, dict(levels=3)),                  # exact-distance ties in both heuristics
    ("ties-cosine", "cosine", 3, 3, 16, 2500, dict(levels=3)),
    ("ties-manhattan", "manhattan", 3, 3, 16, 2500, dict(levels=3)),
    ("dups-manhattan", "manhattan", 8, 4, 10, 2500, dict(dup_frac=0.2)),
    ("d33-cosine", "cosine", 33, 5, 20, 2500, dict(dup_frac=0.1)),     # dims % 4 != 0
    ("d128-l2", "l2", 128, 16, 64, 3000, dict()),
    ("d768-cosine", "cosine", 768, 32, 100, 2500, dict()),             # the bench's metric, row shape and m
    ("m100-ties", "l2", 3, 100, 120, 2500, dict(levels=3)),            # maxM 200 > one warp; a few lists fill and are re-pruned
    ("m1", "l2", 8, 1, 8, 2500, dict()),                               # maxM 2: almost every back-link re-prunes
    ("m0", "manhattan", 5, 0, 8, 2500, dict()),                        # reloption minimum: no links at all
]

# the same bodies on the emulated library (tests/test_capi_emulated.py): n 400 - 500, batches of up to 11 - 15
EMU_CASES = [
    ("l2-d8", "l2", 8, 4, 16, 400, dict()),
    ("ties-l2", "l2", 3, 3, 16, 400, dict(levels=3)),
    ("cosine-d12", "cosine", 12, 4, 16, 500, dict()),
    ("m0", "manhattan", 5, 0, 8, 400, dict()),
    ("m1", "l2", 5, 1, 8, 400, dict()),
]


def cid(c):
    return c[0]


@pytest.fixture(scope="module")
def pg():
    import pg_embedding_b200 as pg
    from pg_embedding_b200 import build
    build.build()
    if pg.device_count() < 1:
        pytest.fail("no CUDA device: the product path has no CPU fallback")
    return pg


def case_data(cfg, nq=48):
    """Rows, queries (the first four are stored rows) and labels != ids of a case, seeded by the case."""
    name, metric, dims, m, efc, n, kw = cfg
    rng = np.random.default_rng(sum(map(ord, name)) + 7 * n)
    x = _data(rng, n, dims, **kw)
    q = _data(rng, nq, dims, **{k: v for k, v in kw.items() if k == "levels"})
    if metric == "cosine":
        x, q = x + 1.0, q + 1.0
    q[:4] = x[:4]
    labels = (rng.permutation(n).astype(np.uint64) << np.uint64(32)) | np.uint64(5)
    return x, q, labels


def check_bulk_build(pg, oracle_mod, cfg, batch_max, plan="one", coop=None, efs=(10, 64)):
    """Build the case on the device and with the model, compare link lists and searches; returns the model's batch sizes.
    plan: "one" = one build_appended(0, n); "two" = build_appended(0, a), append, build_appended(a, n - a); "reserve" = the
    same with the index grown from capacity a to n in between; "insert" = insert_many of the first a rows, then a bulk build
    of the rest.  coop: PGEMB_COOP for the builds ("0" throughput mode only, "1" latency mode for batches up to one per SM)."""
    name, metric, dims, m, efc, n, kw = cfg
    x, q, labels = case_data(cfg)
    a = n * 2 // 5
    model = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=a if plan == "reserve" else n)
    with kernel_mode(coop) if coop is not None else contextlib.nullcontext():
        if plan == "one":
            model.append_unbound(x, labels)
            sizes = model.build_bulk(0, n, batch_max)
            idx.append(x, labels)
            idx.build_appended(0, n, batch_max)
        else:
            if plan == "insert":
                model.build(x[:a], labels[:a])
                idx.insert_many(x[:a], labels[:a])
                sizes = []
            else:
                model.append_unbound(x[:a], labels[:a])
                sizes = model.build_bulk(0, a, batch_max)
                idx.append(x[:a], labels[:a])
                idx.build_appended(0, a, batch_max)
            if plan == "reserve":
                idx.reserve(n)
            model.append_unbound(x[a:], labels[a:])
            sizes += model.build_bulk(a, n - a, batch_max)
            idx.append(x[a:], labels[a:])
            idx.build_appended(a, n - a, batch_max)
    assert sum(sizes) == (n - a if plan == "insert" else n - 1), (name, plan)
    assert max(sizes) <= batch_max and sizes[-1] >= 1
    got, want = idx.links(), model.links()
    bad = np.flatnonzero((got != want).any(1))
    assert bad.size == 0, (name, batch_max, plan, coop, "link lists differ at nodes", bad[:10], got[bad[0]][:8], want[bad[0]][:8])
    assert idx.labels().tobytes() == labels.tobytes()
    g = Graph()
    g.metric, g.x, g.labels, g.orc, g.ref = metric, x, labels, model, None
    if oracle_mod.available("ref"):
        g.ref = oracle_mod.FlatIndex("ref", dims, m, efc, 64, metric, capacity=n)
        g.ref.load_graph(x, want, labels)
    for ef in efs:
        check(idx, oracle_mod, g, q, ef, (name, batch_max, plan, coop, ef))
    idx.close()
    model.close()
    return sizes


def assert_reaches(sizes, batch_max):
    """n >= 2200: batch_max up to 64 is reached, and 4096 gives batches above 64 (the schedule's own bound, pos / 32)."""
    if batch_max <= 64:
        assert max(sizes) == batch_max, (batch_max, max(sizes))
    else:
        assert max(sizes) > 64, max(sizes)
    assert sizes[0] == 1


@pytest.mark.parametrize("batch_max", BATCH_MAX)
@pytest.mark.parametrize("cfg", CASES, ids=cid)
def test_bulk_build_equals_model(pg, oracle_mod, cfg, batch_max):
    assert_reaches(check_bulk_build(pg, oracle_mod, cfg, batch_max), batch_max)


@pytest.mark.parametrize("plan", ["two", "reserve", "insert"])
@pytest.mark.parametrize("cfg", [CASES[1], CASES[3], CASES[9]], ids=cid)
def test_incremental_bulk_builds(pg, oracle_mod, cfg, plan):
    """A second build_appended with first > 0 (the bench's call shape), after a reserve, and after sequential inserts: the first
    batch of the second call is already a / 32 nodes."""
    sizes = check_bulk_build(pg, oracle_mod, cfg, 4096, plan=plan)
    assert max(sizes) > 64


@pytest.mark.parametrize("coop", ["0", "1"])
def test_bulk_build_either_kernel_mode(pg, oracle_mod, coop):
    """PGEMB_COOP=1 (the default) searches batches of up to one node per SM in latency mode and larger ones in throughput mode;
    PGEMB_COOP=0 searches every batch in throughput mode.  Both give the model's graph."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cfg = ("coop-l2-d16", "l2", 16, 8, 40, 6000, dict())
    sizes = check_bulk_build(pg, oracle_mod, cfg, 4096, coop=coop)
    assert min(sizes) <= sms < max(sizes), (sms, max(sizes))


def test_batch_cap_at_bench_scale(pg, oracle_mod):
    """The bench's batch_max = 4096 where it applies: from node 131 072 on, 4096-node batches, long same-target segments in
    backlink_kernel and 4096 x M pairs in the cub sort."""
    cfg = ("cap-l2-d16", "l2", 16, 8, 40, 140_000, dict())
    sizes = check_bulk_build(pg, oracle_mod, cfg, 4096, efs=(64,))
    starts = np.cumsum([1] + sizes[:-1])
    capped = np.flatnonzero(np.array(sizes) == 4096)
    assert capped.size == 2 and starts[capped[0] - 1] < 131_072 <= starts[capped[0]], (capped.size, starts[capped[:1]])
