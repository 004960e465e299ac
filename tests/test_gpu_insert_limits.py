"""GPU tests of the insert path (csrc/bind_kernel.cuh: the raw-mode traversal, select_kernel, backlink_kernel) at the edges of
its fixed-size structure, byte for byte against the oracle.

The reference accepts m up to what a page holds (maxM 2036 at 1-d) and any efConstruction >= 1; the other device tests stay at
maxM <= 200 and efConstruction <= 300.  Each case here crosses one boundary that the kernels' constants and size formulas
define (mirrored below, never bare numbers), and asserts that it reached it:
- a full list's candidate set C1 = maxM + 1 above the CTA's threads (backlink_kernel's scoring, rank and scan-order loops):
  m = 127 / 128 / 129 on a 3-d integer grid, whose ties and duplicates fill lists;
- kept sets longer than one pass of NG = 256 / LANES row groups, with candidates that only a row kept after the first NG
  rejects (copies of two points);
- the staged select's 256-entry kept_norm table and its M <= 256 gate: m = 256 (staged, 256 rows kept) against 257 (unstaged);
- backlink_kernel's shared memory above 48 KB and traversal hops of more than 512 ids: m = 900;
- efConstruction across the select's thread count, its 48 KB attribute path, the traversal's global-memory result queues and
  the CTA's opt-in shared memory, where select_global_kernel takes over;
- inserts into a graph with deleted nodes (searchBaseLayer ignores the flag, and so must raw mode).

Link lists equal the oracle's (the C restatement `port` and, when it travelled with the tree, the compiled reference `ref`),
and searches of the finished graph equal the oracle's: labels, traversal counters and distance bits (`check` of
tests/test_gpu_visited_set.py).  tests/test_capi_emulated.py runs the replay, kept-set, efConstruction and deleted-node
bodies on the host-emulated library at smaller n."""
import contextlib
import functools
import json
import os
import re
import tempfile

import numpy as np
import pytest

from test_gpu_parity import _data, kernel_mode
from test_gpu_visited_set import Graph, check

pytestmark = pytest.mark.gpu

# ---- the kernels' constants and size formulas, mirrored ----------------------------------------------------------------
BIND_THREADS = 256                                   # kBindThreads (bind_kernel.cuh)
LANES = {"l2": 8, "cosine": 4, "manhattan": 4}       # MetricLanes (dist_exact.cuh)
MAX_CTA_SMEM = 232448                                # kMaxCtaSmem (search_config.h): the H100's opt-in per CTA
DEFAULT_SMEM = 48 * 1024                             # above this a launch needs cudaFuncSetAttribute
STAGED_KEPT = 256                                    # heuristic_block_staged's kept_norm[] and launch_connect's M gate
SMEM_VISITED = 1024                                  # the smallest latency-mode visited table (make_search_config)


def row_groups(metric):
    """NG of heuristic_block: kept rows tested per pass."""
    return BIND_THREADS // LANES[metric]


def select_smem(efc, m):
    """select_smem_bytes(ef, M, row_f, staged=false): candidate keys, kept keys, scan order."""
    return efc * 8 + max(m, 1) * 8 + efc * 4


def select_global_smem(m):
    """select_global_smem_bytes(M): the kept keys only."""
    return max(m, 1) * 8


def backlink_smem(maxm):
    """launch_backlinks: two key arrays of maxM + 1, the kept keys, the scan order."""
    return (maxm + 1) * 8 * 2 + max(maxm, 1) * 8 + (maxm + 1) * 4


def res_global_ef():
    """The smallest ef whose two result queues (2 x ef x 8 bytes) exceed a CTA (make_search_config returns 1)."""
    return MAX_CTA_SMEM // 16 + 1


def efc_select_above(limit, m):
    """The smallest efConstruction whose select_kernel needs more than `limit` bytes."""
    return (limit - max(m, 1) * 8) // 12 + 1


@pytest.fixture(scope="module")
def pg():
    import pg_embedding_b200 as pg
    from pg_embedding_b200 import build
    build.build()
    if pg.device_count() < 1:
        pytest.fail("no CUDA device: the product path has no CPU fallback")
    return pg


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def bind_launches(run):
    """Runs `run()`; returns [(kernel name or None, threads per CTA, dynamic shared memory or None)] of its launches.  On a
    device from torch.profiler's CUDA trace (names such as "select_global_kernel<2>"); on the emulated library from its
    runtime's launch log (no names, but every launch's dynamic shared memory)."""
    import ctypes as C
    import torch
    if torch.cuda.is_available():
        from torch.profiler import ProfilerActivity, profile
        with tempfile.TemporaryDirectory() as tmp:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            path = os.path.join(tmp, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                events = json.load(f)["traceEvents"]
        out = []
        for e in events:
            if e.get("cat") == "kernel":
                m = re.search(r"pgemb::(\w+(?:<[^>]*>)?)", e["name"])     # "void pgemb::select_kernel<1, true>(pgemb::GraphView, ...)"
                out.append((m[1] if m else e["name"], int(e["args"]["block"][0]), e["args"].get("shared memory")))
        return out
    from pg_embedding_b200 import _lib
    lib = _lib.load()
    cap = 4096
    threads, smem = (C.c_uint * cap)(), (C.c_size_t * cap)()
    lib.emu_launch_log.argtypes = [C.POINTER(C.c_uint), C.POINTER(C.c_size_t), C.c_int]
    lib.emu_launch_log(threads, smem, cap)
    run()
    k = lib.emu_launch_log(threads, smem, cap)
    return [(None, int(threads[i]), int(smem[i])) for i in range(min(k, cap))]


def assert_select_path(launches, efc, m, what):
    """The select of these launches ran in shared memory below the opt-in limit and from the workspace above it."""
    glob = select_smem(efc, m) > MAX_CTA_SMEM
    names = [l[0] for l in launches if l[0] is not None]
    if names:
        sel = [nm for nm in names if nm.startswith("select_")]
        assert sel, (what, names[:8])
        assert all(nm.startswith("select_global_kernel" if glob else "select_kernel") for nm in sel), (what, efc, sel[:4])
        return
    sizes = [s for _, t, s in launches if t == BIND_THREADS]
    assert all(s <= MAX_CTA_SMEM for _, _, s in launches), (what, max(s for _, _, s in launches))
    if glob:
        assert select_global_smem(m) in sizes and select_smem(efc, m) not in sizes, (what, efc, sorted(set(sizes)))
    else:   # select_kernel, staged (its rows behind the keys) or not
        assert any(s >= select_smem(efc, m) for s in sizes), (what, efc, sorted(set(sizes)))


def oracles(oracle_mod):
    return ["port"] + (["ref"] if oracle_mod.available("ref") else [])


def diff_nodes(got, want):
    return np.flatnonzero((got != want).any(1))


def assert_links(got, want, what):
    bad = diff_nodes(got, want)
    assert bad.size == 0, (what, "link lists differ at nodes", bad[:10], got[bad[0]][:8], want[bad[0]][:8])


def search_graph(oracle_mod, metric, dims, m, efc, x, links, nq=64, levels=0, seed=0):
    """A Graph for `check`: the oracle(s) holding this graph and nq queries (the first four are stored rows)."""
    n = x.shape[0]
    rng = np.random.default_rng(seed)
    g = Graph()
    g.metric, g.x = metric, x
    g.q = _data(rng, nq, dims, levels=levels) + (1.0 if metric == "cosine" else 0.0)
    g.q[:4] = x[:4]
    g.labels = np.arange(n, dtype=np.uint64)
    g.orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    g.orc.load_graph(x, links, g.labels)
    g.ref = None
    if oracle_mod.available("ref"):
        g.ref = oracle_mod.FlatIndex("ref", dims, m, efc, 64, metric, capacity=n)
        g.ref.load_graph(x, links, g.labels)
    return g


def check_search_modes(pg, oracle_mod, idx, g, ef, what, smem_visited=False):
    """Search parity in latency mode (optionally with the smallest shared-memory visited table) and in throughput mode."""
    visits = []
    for coop in ("1", "0"):
        knobs = {"PGEMB_SMEM_VISITED": SMEM_VISITED} if (smem_visited and coop == "1") else {}
        with kernel_mode(coop), env(**knobs):
            visits.append(check(idx, oracle_mod, g, g.q, ef, (what, "coop", coop))[0])
    return visits


# ---- m = 127 / 128 / 129: full lists re-pruned with C1 = 255 / 257 / 259 ------------------------------------------------
@functools.lru_cache(maxsize=None)
def grid_build(oracle_mod, which, m, metric, n, replay, efc=300):
    """The oracle's build of a 2-level 3-d grid, with the records before the last `replay` inserts, and for each of those
    inserts the largest list it took a back-link into when that list was already full (0 = none)."""
    rng = np.random.default_rng(m * 7 + n)
    x = _data(rng, n, 3, levels=2) + (1.0 if metric == "cosine" else 0.0)
    cut = n - replay
    orc = oracle_mod.FlatIndex(which, 3, m, efc, 64, metric, capacity=n)
    orc.build(x[:cut])
    before = orc.records().copy()
    full_hits = 0
    for i in range(cut, n):
        prev = orc.links()
        orc.add(x[i], i)
        own = orc.links(i, 1)[0]
        tgt = own[1:1 + own[0]]
        full_hits += int((prev[tgt, 0] == 2 * m).sum())
    return x, before, orc.links(), full_hits


def check_full_lists(pg, oracle_mod, m, metric, n, replay, full_build):
    """The last `replay` inserts on the device from the oracle's records before them (and, with full_build, the whole build by
    insert_many): link lists equal the oracle's, and those inserts re-pruned full lists of maxM + 1 candidates."""
    names = oracles(oracle_mod)
    builds = {w: grid_build(oracle_mod, w, m, metric, n, replay) for w in names}
    x, before, want, hits = builds[names[-1]]
    for w in names[:-1]:
        assert_links(builds[w][2], want, (m, metric, w, "oracles disagree"))
    assert hits > 0, (m, metric, "no back-link reached a full list")
    assert want[:, 0].max() == 2 * m
    idx = pg.HnswIndex(3, m, 300, 64, metric, capacity=n)
    idx.load_records(before)
    idx.insert_many(x[n - replay:])
    assert_links(idx.links(), want, (m, metric, "replay"))
    idx.close()
    if full_build:
        idx = pg.HnswIndex(3, m, 300, 64, metric, capacity=n)
        idx.insert_many(x)
        assert_links(idx.links(), want, (m, metric, "full build"))
        g = search_graph(oracle_mod, metric, 3, m, 300, x, want, levels=2, seed=m)
        check_search_modes(pg, oracle_mod, idx, g, 64, (m, metric))
        idx.close()
    return hits


FULL_LIST_CASES = [(m, metric) for m in (127, 128, 129) for metric in ("l2", "cosine", "manhattan")]


@pytest.mark.parametrize("m,metric", FULL_LIST_CASES,
                         ids=[f"C1-{2 * m + 1}-{'below' if 2 * m + 1 < BIND_THREADS else 'above'}-threads-{mt}" for m, mt in FULL_LIST_CASES])
def test_full_list_repruning_across_threads(pg, oracle_mod, m, metric):
    """C1 = maxM + 1 below (255), just above (257) and two above (259) backlink_kernel's 256 threads; more than NG rows kept."""
    assert (2 * m + 1 > BIND_THREADS) == (m >= 128)
    assert 2 * m > row_groups(metric)
    check_full_lists(pg, oracle_mod, m, metric, 2500, 300, full_build=(metric == "l2"))


# ---- kept sets beyond one pass of NG row groups, with rejections decided by a later row ---------------------------------
def check_kept_beyond_row_groups(pg, oracle_mod, metric, n):
    """M = NG + 16 and rows that are mostly copies of two points A and B, efConstruction = n.  A copy of A keeps every earlier
    copy of A (distance 0 to it) -- more than NG once enough exist, fewer than M -- then B's first copy; every further copy of
    B is rejected only by that first one, which sits beyond the first NG kept rows.  A heuristic that tested fewer kept rows
    would keep those copies."""
    ng = row_groups(metric)
    m, dims = ng + 16, 6
    rng = np.random.default_rng(ng + n)
    x = rng.standard_normal((n, dims)).astype(np.float32) + (1.0 if metric == "cosine" else 0.0)
    x[16:] = x[rng.integers(0, 2, n - 16)]
    want = None
    for w in oracles(oracle_mod):
        orc = oracle_mod.FlatIndex(w, dims, m, n, 64, metric, capacity=n)
        orc.build(x)
        if want is None:
            want = orc.links()
        assert_links(orc.links(), want, (metric, w, "oracles disagree"))
        orc.close()
    assert (want[:, 0] > ng).sum() > n // 4, (ng, np.bincount(want[:, 0])[ng:])
    for staged in ("1", "0"):
        with env(PGEMB_SELECT_STAGED=staged):
            idx = pg.HnswIndex(dims, m, n, 64, metric, capacity=n)
            idx.insert_many(x)
            assert_links(idx.links(), want, (metric, "staged", staged))
            idx.close()


@pytest.mark.parametrize("metric", ["l2", "cosine", "manhattan"])
def test_kept_set_beyond_row_groups(pg, oracle_mod, metric):
    check_kept_beyond_row_groups(pg, oracle_mod, metric, 600)


# ---- m = 256 / 257: the staged select keeps 256 rows; one more takes the unstaged kernel -----------------------------
def dup_rows(n, dims, seed):
    """Cosine rows in which all but the first 100 are copies of row 0: a copy's candidates at distance 0 are all kept."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, dims)).astype(np.float32) + 1.0
    x[100:] = x[0]
    return x


@pytest.mark.parametrize("m", [STAGED_KEPT, STAGED_KEPT + 1], ids=["staged-kept-256", "unstaged-m257"])
def test_wide_select_staged_gate(pg, oracle_mod, m):
    n, dims, efc = 2 * m + 100, 8, 2 * m + 100
    x = dup_rows(n, dims, m)
    want = None
    for w in oracles(oracle_mod):
        orc = oracle_mod.FlatIndex(w, dims, m, efc, 64, "cosine", capacity=n)
        orc.build(x)
        if want is None:
            want = orc.links()
        assert_links(orc.links(), want, (m, w, "oracles disagree"))
        orc.close()
    assert want[n - 1, 0] == m                      # the last copy kept M rows (its own list, untouched since)
    assert (want[:, 0] == 2 * m).any()              # and full lists were re-pruned with C1 = 2m + 1 candidates
    # insert(): one bind per launch, the staged select for M <= 256
    idx = pg.HnswIndex(dims, m, efc, 64, "cosine", capacity=n)
    idx.insert_many(x[:n - 4])
    launches = bind_launches(lambda: [idx.insert(x[i]) for i in range(n - 4, n)])
    assert_links(idx.links(), want, (m, "insert"))
    names = [l[0] for l in launches if l[0] and l[0].startswith("select_")]
    if names:
        assert all(("true" in nm) == (m <= STAGED_KEPT) for nm in names), names
    idx.close()
    with env(PGEMB_SELECT_STAGED=0):
        idx = pg.HnswIndex(dims, m, efc, 64, "cosine", capacity=n)
        idx.insert_many(x)
        assert_links(idx.links(), want, (m, "unstaged"))
        idx.close()


# ---- m = 900: backlink_kernel above 48 KB, hops of more than 512 ids ---------------------------------------------------
def test_maxm_1800_backlinks_and_wide_hops(pg, oracle_mod):
    m, efc, n, dims = 900, 1000, 2000, 2
    assert backlink_smem(2 * m) > DEFAULT_SMEM
    rng = np.random.default_rng(900)
    x = _data(rng, n, dims, levels=40)
    want = None
    for w in oracles(oracle_mod):
        orc = oracle_mod.FlatIndex(w, dims, m, efc, 64, "l2", capacity=n)
        orc.build(x)
        if want is None:
            want = orc.links()
        assert_links(orc.links(), want, ("m900", w, "oracles disagree"))
        orc.close()
    assert (want[:, 0] > SMEM_VISITED // 2).sum() > 10, want[:, 0].max()
    idx = pg.HnswIndex(dims, m, efc, 64, "l2", capacity=n)
    idx.insert_many(x)
    assert_links(idx.links(), want, "m900")
    g = search_graph(oracle_mod, "l2", dims, m, efc, x, want, levels=40, seed=9)
    lat, thr = check_search_modes(pg, oracle_mod, idx, g, 64, "m900", smem_visited=True)
    assert (lat > SMEM_VISITED // 2).any() and (lat == thr).all()    # the shared-memory table migrated within a hop
    idx.close()


# ---- efConstruction across the select's and the traversal's shared-memory limits --------------------------------------
EFC_M = 8
EFC_CASES = [("efc-above-threads", BIND_THREADS + 1, "l2"),
             ("efc-select-above-48k", efc_select_above(DEFAULT_SMEM, EFC_M), "cosine"),
             ("efc-search-results-global", res_global_ef(), "manhattan"),
             ("efc-select-above-optin", efc_select_above(MAX_CTA_SMEM, EFC_M), "l2")]


def check_efc(pg, oracle_mod, efc, metric, n, dims=8, batch_max=64):
    """Every bind path at this efConstruction: hnsw_bind_point (insert), insert_many, build(batch_max=1), the bulk build against
    the oracle's batch model and the exact parallel build."""
    rng = np.random.default_rng(efc)
    x = rng.standard_normal((n, dims)).astype(np.float32) + (1.0 if metric == "cosine" else 0.0)
    want = None
    for w in oracles(oracle_mod):
        orc = oracle_mod.FlatIndex(w, dims, EFC_M, efc, 64, metric, capacity=n)
        orc.build(x)
        if want is None:
            want = orc.links()
        assert_links(orc.links(), want, (efc, w, "oracles disagree"))
        orc.close()
    half = n // 2
    idx = pg.HnswIndex(dims, EFC_M, efc, 64, metric, capacity=n)
    idx.insert_many(x[:half])
    for i in range(half, half + 5):
        idx.insert(x[i])
    launches = bind_launches(lambda: idx.insert_many(x[half + 5:]))
    assert_links(idx.links(), want, (efc, "insert / insert_many"))
    assert_select_path(launches, efc, EFC_M, efc)
    idx.close()
    idx = pg.HnswIndex(dims, EFC_M, efc, 64, metric, capacity=n)
    with kernel_mode("0"):
        idx.build(x, batch_max=1)
    assert_links(idx.links(), want, (efc, "build(batch_max=1)"))
    idx.close()
    model = oracle_mod.FlatIndex("port", dims, EFC_M, efc, 64, metric, capacity=n)
    model.append_unbound(x)
    sizes = model.build_bulk(0, n, batch_max)
    assert max(sizes) > 1
    idx = pg.HnswIndex(dims, EFC_M, efc, 64, metric, capacity=n)
    idx.append(x)
    idx.build_appended(0, n, batch_max)
    assert_links(idx.links(), model.links(), (efc, "bulk build"))
    idx.close()
    model.close()
    idx = pg.HnswIndex(dims, EFC_M, efc, 64, metric, capacity=n)
    idx.append(x)
    idx.build_exact(0, n, 256)
    assert_links(idx.links(), want, (efc, "exact build"))
    idx.close()


@pytest.mark.parametrize("case", EFC_CASES, ids=[c[0] for c in EFC_CASES])
def test_efconstruction_ladder(pg, oracle_mod, case):
    name, efc, metric = case
    check_efc(pg, oracle_mod, efc, metric, 2500)


# ---- deleted nodes: the bind's search expands and links them ------------------------------------------------------------
def check_deleted(pg, oracle_mod, metric, n, dims=8, m=8, efc=40):
    """A third of the first half marked deleted before the second half is inserted: same lists as the reference, whose
    searchBaseLayer ignores the flag, and the new lists do name deleted nodes."""
    rng = np.random.default_rng(31 + n)
    x = _data(rng, n, dims) + (1.0 if metric == "cosine" else 0.0)
    half = n // 2
    dead = np.arange(0, half, 3)
    want = None
    for w in oracles(oracle_mod):
        orc = oracle_mod.FlatIndex(w, dims, m, efc, 64, metric, capacity=n)
        orc.build(x[:half])
        for i in dead:
            orc.mark_deleted(int(i))
        for i in range(half, n):
            orc.add(x[i], i)
        if want is None:
            want = orc.links()
        assert_links(orc.links(), want, (metric, w, "oracles disagree"))
        orc.close()
    new = want[half:]
    named = [np.isin(r[1:1 + r[0]], dead).any() for r in new]
    assert sum(named) > len(new) // 4, sum(named)
    idx = pg.HnswIndex(dims, m, efc, 64, metric, capacity=n)
    idx.insert_many(x[:half])
    idx.mark_deleted(dead)
    idx.insert_many(x[half:])
    assert_links(idx.links(), want, (metric, "deleted"))
    idx.close()


@pytest.mark.parametrize("metric", ["l2", "cosine", "manhattan"])
def test_insert_into_graph_with_deleted_nodes(pg, oracle_mod, metric):
    check_deleted(pg, oracle_mod, metric, 3000)
