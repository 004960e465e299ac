"""search_kernel -- the traversal itself, throughput mode (a warp per query, ring pool, bulk-TMA gathers) and latency
mode (a CTA per query) -- executed on the HOST by the SIMT emulator in tests/emu and compared with the oracle: same
labels, same order, same per-query traversal counters.  Checks the kernel's logic (queue update, visited set,
ring-pool and mbarrier protocol, emit order) without a GPU; the `-m gpu` tests remain the parity tests proper."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest



def sqnorm_lane_order(v):
    """|v|^2 in the cosine lane order (4 lane-strided partial sums, (s0+s2)+(s1+s3), scalar tail): distfunc.c:141-142 as built."""
    v = v.astype(np.float32)
    main = v.size & ~3
    s = np.zeros(4, np.float32)
    for i in range(0, main, 4):
        s = s + v[i:i + 4] * v[i:i + 4]
    res = np.float32(np.float32(s[0] + s[2]) + np.float32(s[1] + s[3]))
    for e in range(main, v.size):
        res = np.float32(res + np.float32(v[e] * v[e]))
    return res

# the emulated CTAs are real threads: a protocol bug could hang them -- fail the run instead of blocking it
pytestmark = pytest.mark.timeout(900, method="thread")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRIC_ID = {"l2": 0, "cosine": 1, "manhattan": 2}


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


@pytest.fixture(autouse=True, params=["issue", "late"], ids=["tma-at-issue", "tma-late"])
def tma_schedule(request, monkeypatch):
    """Every test runs under the two extreme legal completion times of a bulk copy: performed when issued, or only when
    its mbarrier is polled (a consumer that does not wait -- or waits on the wrong barrier / parity -- fails under "late")."""
    monkeypatch.setenv("PGEMB_EMU_TMA", request.param)
    return request.param


def _build_emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "libsearch_emu.so")
    src = [os.path.join(ROOT, "tests", "emu", f) for f in ("search_emu.cpp", "emu_runtime.cpp")]
    cmd = ["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I", os.path.join(ROOT, "tests", "emu", "fake_cuda"), "-o", out] + src
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lib = C.CDLL(out)
    lib.emu_search.restype = C.c_int
    lib.emu_search_ex.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """The kernels as the product library compiles them."""
    return _build_emu(tmp_path_factory)


@pytest.fixture(scope="module")
def emu_proto(emu):
    """Round 1 kept the then-unmeasured variants (paired visited test, shared-memory visited set, 8 lanes per L2 row) in a
    separate -DPGEMB_PROTO build; they are product code now, so this is the same library."""
    return emu


def run_emu(lib, metric, coop, x, links, labels, q, ef, maxm, warps, rings, grid, vh, pairs=0, smem_visited=0, tpr8=False, resg=False):
    n, dim = x.shape
    row_f = (dim + 3) & ~3
    ls = (maxm + 1 + 3) & ~3
    xv = np.zeros((n, row_f), np.float32); xv[:, :dim] = x
    lk = np.zeros((n, ls), np.uint32); lk[:, :maxm + 1] = links
    norms = np.array([sqnorm_lane_order(x[i]) for i in range(n)], np.float32) if metric == "cosine" else np.zeros(n, np.float32)
    nq = q.shape[0]
    lab = np.zeros((nq, ef), np.uint64); dd = np.zeros((nq, ef), np.float32); ids = np.zeros((nq, ef), np.uint32)
    nn = np.zeros(nq, np.int32); st = np.zeros((nq, 4), np.uint32)
    err = C.c_int(0)
    rc = lib.emu_search_ex(METRIC_ID[metric], coop, _p(xv, C.c_float), _p(lk, C.c_uint32), _p(labels, C.c_uint64), _p(norms, C.c_float),
                        C.c_uint32(n), C.c_uint32(dim), C.c_uint32(row_f), C.c_uint32(ls), C.c_uint32(maxm), _p(np.ascontiguousarray(q), C.c_float),
                        C.c_uint32(nq), C.c_uint32(ef), 0, _p(lab, C.c_uint64), _p(dd, C.c_float), _p(ids, C.c_uint32), _p(nn, C.c_int32),
                        _p(st, C.c_uint32), C.c_uint32(warps), C.c_uint32(rings), C.c_uint32(grid), C.c_uint32(vh), C.c_uint32(pairs), C.c_uint32(smem_visited | (0x80000000 if tpr8 else 0) | (0x20000000 if resg else 0)), C.byref(err))
    assert rc == 0, rc
    assert err.value == 0, hex(err.value)
    assert lib.emu_tma_unwaited() == 0, "a bulk copy was still in flight when its CTA exited"
    return dict(labels=lab, dists=dd, ids=ids, n=nn, stats=st)


CASES = [
    # metric, dims, m, efC, n, levels, ef, nq
    ("l2", 3, 3, 16, 120, 3, 5, 6),          # tie-heavy (integer grid): overflow list, equal-distance pops
    ("cosine", 16, 4, 20, 300, 0, 8, 8),
    ("manhattan", 33, 5, 20, 250, 0, 12, 6),  # dims % 4 != 0: padded rows, scalar tails
    ("l2", 40, 20, 24, 200, 0, 16, 5),       # maxM = 40: more than one 32-id chunk per link list, 5 row groups per hop
    ("cosine", 24, 50, 16, 260, 0, 10, 4),   # maxM = 100: four 32-id chunks per link list, 13 row groups per hop
]


@pytest.mark.parametrize("pairs", [0, 1], ids=["ordered-visited", "paired-visited"])
@pytest.mark.parametrize("coop", [0, 1], ids=["throughput", "latency"])
@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-d{c[1]}m{c[2]}" for c in CASES])
def test_search_kernel_emulated_matches_oracle(emu, emu_proto, oracle_mod, case, coop, pairs):
    emu = emu_proto if pairs else emu
    metric, dims, m, efc, n, levels, ef, nq = case
    rng = np.random.default_rng(31 + dims)
    if levels:
        x = rng.integers(0, levels, (n, dims)).astype(np.float32); q = rng.integers(0, levels, (nq, dims)).astype(np.float32)
    else:
        x = rng.standard_normal((n, dims)).astype(np.float32); q = rng.standard_normal((nq, dims)).astype(np.float32)
    if metric == "cosine":
        x, q = x + 1.0, q + 1.0
    labels = (rng.permutation(n).astype(np.uint64) << np.uint64(20)) | np.uint64(3)
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    orc.build(x, labels)
    for i in range(0, n, 7):
        orc.mark_deleted(i)
    links, labs = orc.links(), orc.labels()
    want = orc.search_many(q, ef, want_counters=True)
    # throughput mode: 3 slots share 2 rings on 2 "SMs" (lock contention + work stealing); latency mode: a CTA per query;
    # a 64-entry hash visited set forces the migration to the bitmap on the larger graphs
    got = run_emu(emu, metric, coop, x, links, labs, q, ef, 2 * m, warps=3, rings=2, grid=2, vh=64, pairs=pairs)
    assert got["n"].tolist() == want["n"].tolist()
    assert got["labels"].tobytes() == want["labels"].tobytes()
    assert got["stats"][:, :3].tolist() == want["counters"][:, :3].tolist()
    for qi in range(nq):
        k = int(got["n"][qi])
        dref = oracle_mod.dist_many("port", metric, q[qi], x[got["ids"][qi, :k]]) if k else np.zeros(0, np.float32)
        assert got["dists"][qi, :k].tobytes() == dref.tobytes()


@pytest.mark.parametrize("coop", [0, 1], ids=["throughput", "latency"])
def test_search_kernel_emulated_very_large_ef(emu, oracle_mod, coop):
    """efSearch in the thousands (the scan doubles it for large LIMITs, embedding.c:334): queues far larger than the graph."""
    rng = np.random.default_rng(77)
    n, dims, m = 500, 12, 6
    x = rng.standard_normal((n, dims)).astype(np.float32)
    q = rng.standard_normal((3, dims)).astype(np.float32)
    orc = oracle_mod.FlatIndex("port", dims, m, 24, 64, "l2", capacity=n)
    orc.build(x)
    for ef in (300, 6000):
        want = orc.search_many(q, ef, want_counters=True)
        got = run_emu(emu, "l2", coop, x, orc.links(), orc.labels(), q, ef, 2 * m, warps=2, rings=2, grid=2, vh=64)
        assert got["n"].tolist() == want["n"].tolist()
        assert got["labels"].tobytes() == want["labels"].tobytes()
        assert got["stats"][:, :3].tolist() == want["counters"][:, :3].tolist()


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-d{c[1]}m{c[2]}" for c in CASES])
def test_result_queues_in_global_memory(emu, oracle_mod, case):
    """search_kernel<..., RESG>: the variant plan_search falls back to when 2 x ef keys do not fit shared memory (no ef ceiling:
    the reference doubles efSearch without bound, embedding.c:334).  Same labels, distances and traversal counters, incl. an ef
    far above the number of nodes."""
    metric, dims, m, efc, n, levels, ef, nq = case
    rng = np.random.default_rng(77 + dims)
    if levels:
        x = rng.integers(0, levels, (n, dims)).astype(np.float32); q = rng.integers(0, levels, (nq, dims)).astype(np.float32)
    else:
        x = rng.standard_normal((n, dims)).astype(np.float32); q = rng.standard_normal((nq, dims)).astype(np.float32)
    if metric == "cosine":
        x, q = x + 1.0, q + 1.0
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    orc.build(x)
    for e in (ef, 5 * n):
        want = orc.search_many(q, e, want_counters=True)
        got = run_emu(emu, metric, 0, x, orc.links(), orc.labels(), q, e, 2 * m, warps=3, rings=2, grid=2, vh=64, resg=True)
        assert got["n"].tolist() == want["n"].tolist() and got["labels"].tobytes() == want["labels"].tobytes()
        assert got["stats"][:, :3].tolist() == want["counters"][:, :3].tolist()


BIND_CASES = [
    # metric, dims, m, efC, n, levels
    ("l2", 3, 3, 8, 70, 3),          # ties + duplicates: equal-distance scan order of the heuristic, full lists re-pruned
    ("cosine", 16, 4, 12, 60, 0),
    ("manhattan", 9, 2, 6, 50, 0),   # M = 2, maxM = 4: lists fill quickly, re-prune path on most inserts
]


@pytest.mark.parametrize("coop", [0, 1], ids=["throughput", "latency"])
@pytest.mark.parametrize("case", BIND_CASES, ids=[f"{c[0]}-d{c[1]}m{c[2]}" for c in BIND_CASES])
def test_bind_kernels_emulated_match_oracle(emu, oracle_mod, case, coop):
    """n x hnsw_bind_point on the emulator (traversal in raw mode + select_kernel + backlink_kernel per insert):
    every link list must equal the oracle's after the same inserts."""
    metric, dims, m, efc, n, levels = case
    rng = np.random.default_rng(77 + dims)
    x = rng.integers(0, levels, (n, dims)).astype(np.float32) if levels else rng.standard_normal((n, dims)).astype(np.float32)
    if metric == "cosine":
        x = x + 1.0
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
    orc.build(x)
    want = orc.links()
    maxm = 2 * m
    row_f = (dims + 3) & ~3
    ls = (maxm + 1 + 3) & ~3
    xv = np.zeros((n, row_f), np.float32); xv[:, :dims] = x
    lk = np.zeros((n, ls), np.uint32)
    norms = np.array([sqnorm_lane_order(x[i]) for i in range(n)], np.float32) if metric == "cosine" else np.zeros(n, np.float32)
    err = C.c_int(0)
    rc = emu.emu_bind_sequence(METRIC_ID[metric], coop, _p(xv, C.c_float), _p(lk, C.c_uint32), _p(norms, C.c_float), C.c_uint32(n), C.c_uint32(dims),
                               C.c_uint32(row_f), C.c_uint32(ls), C.c_uint32(m), C.c_uint32(maxm), C.c_uint32(efc), C.c_uint32(0), C.c_uint32(n), C.byref(err))
    assert rc == 0 and err.value == 0, (rc, err.value)
    got = lk[:, :maxm + 1]
    bad = np.flatnonzero((got != want).any(1))
    assert bad.size == 0, f"link lists differ at nodes {bad[:8]}: {got[bad[0]]} vs {want[bad[0]]}"


@pytest.mark.parametrize("n,ef", [(300, 12), (1500, 220)], ids=["small", "migrates-to-bitmap"])
def test_latency_mode_shared_memory_visited_set(emu_proto, oracle_mod, n, ef):
    emu = emu_proto
    """Prototype (PGEMB_SMEM_VISITED): in latency mode the open-addressing visited set lives in the CTA's shared memory.
    The 1500-node case visits more than half of the 1024-entry table, so it also crosses the migration to the bitmap."""
    rng = np.random.default_rng(n)
    dims, m, efc = 12, 6, 24
    x = rng.standard_normal((n, dims)).astype(np.float32)
    q = rng.standard_normal((3, dims)).astype(np.float32)
    orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, "l2", capacity=n)
    orc.build(x)
    want = orc.search_many(q, ef, want_counters=True)
    got = run_emu(emu, "l2", 1, x, orc.links(), orc.labels(), q, ef, 2 * m, warps=2, rings=2, grid=2, vh=64, smem_visited=1024)
    assert got["labels"].tobytes() == want["labels"].tobytes()
    assert got["stats"][:, :3].tolist() == want["counters"][:, :3].tolist()
    if n >= 1500:
        assert int(want["counters"][:, 0].max()) > 512, "case too small to cross the half-full migration"


@pytest.mark.parametrize("jitter", ["0", "1"], ids=["", "jitter"])
def test_fuzz_traversal_emulated(emu, emu_proto, oracle_mod, jitter, monkeypatch):
    monkeypatch.setenv("PGEMB_EMU_JITTER", jitter)   # 1: warps pause at random around atomics (ring-pool hand-overs, work stealing meet in many orders)
    """300 seeded random configurations (metric, dims, m, ef, graph size, ties/duplicates, deleted labels, kernel mode,
    slots/rings/CTAs, visited-table size): labels, counts and traversal counters must equal the oracle's every time."""
    for seed in range(300):
        rng = np.random.default_rng(9000 + seed)
        metric = ["l2", "cosine", "manhattan"][rng.integers(0, 3)]
        dims = int(rng.choice([1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 31, 33, 48]))
        m = int(rng.choice([1, 2, 3, 4, 6, 9, 17]))
        efc = int(rng.choice([1, 2, 5, 8, 16, 30]))
        n = int(rng.choice([1, 2, 3, 10, 40, 90, 180]))
        levels = int(rng.choice([0, 0, 2, 3, 5]))
        ef = int(rng.choice([1, 2, 3, 5, 9, 16, 40]))
        nq = int(rng.choice([1, 3, 7]))
        coop = int(rng.integers(0, 2))
        warps, rings, grid = int(rng.choice([1, 2, 3, 4])), int(rng.choice([1, 2, 3])), int(rng.choice([1, 2, 3]))
        vh = int(rng.choice([0, 16, 64, 256]))
        if levels:
            x = rng.integers(0, levels, (n, dims)).astype(np.float32); q = rng.integers(0, levels, (nq, dims)).astype(np.float32)
        else:
            x = rng.standard_normal((n, dims)).astype(np.float32); q = rng.standard_normal((nq, dims)).astype(np.float32)
        if metric == "cosine":
            x, q = x + 1.0, q + 1.0
        if rng.random() < 0.3 and n > 3:
            k = max(1, n // 4)
            x[rng.integers(0, n, k)] = x[rng.integers(0, n, k)]
        labels = (rng.permutation(n).astype(np.uint64) << np.uint64(8)) | np.uint64(1)
        orc = oracle_mod.FlatIndex("port", dims, m, efc, 64, metric, capacity=n)
        orc.build(x, labels)
        for i in range(0, n, 5):
            if rng.random() < 0.5:
                orc.mark_deleted(i)
        want = orc.search_many(q, ef, want_counters=True)
        pairs, sv = int(rng.integers(0, 2)), int(rng.choice([0, 1024]))
        rng.integers(0, 2)      # (keeps the stream of the seeded cases: this draw once chose the removed LDGSTS gather, then the removed row pool)
        sv = sv if coop else 0
        got = run_emu(emu, metric, coop, x, orc.links(), orc.labels(), q, ef, 2 * m, warps=warps, rings=rings, grid=grid, vh=vh, pairs=pairs, smem_visited=sv)
        what = (seed, pairs, sv, metric, dims, m, efc, n, levels, ef, nq, coop, warps, rings, grid, vh)
        assert got["n"].tolist() == want["n"].tolist(), what
        assert got["labels"].tobytes() == want["labels"].tobytes(), what
        assert got["stats"][:, :3].tolist() == want["counters"][:, :3].tolist(), what
        orc.close()


@pytest.mark.parametrize("coop", [0, 1], ids=["throughput", "latency"])
@pytest.mark.parametrize("dims,m,n,levels", [(3, 3, 120, 3), (40, 20, 200, 0), (100, 6, 150, 0), (16, 4, 90, 2)])
def test_l2_eight_lanes_per_row(emu_proto, oracle_mod, dims, m, n, levels, coop):
    emu = emu_proto
    """Prototype (PGEMB_L2_TPR8): L2 rows scored by 8 lanes, one reference accumulator lane each, rings of 4 rows."""
    rng = np.random.default_rng(dims * 3 + n)
    x = rng.integers(0, levels, (n, dims)).astype(np.float32) if levels else rng.standard_normal((n, dims)).astype(np.float32)
    q = rng.integers(0, levels, (5, dims)).astype(np.float32) if levels else rng.standard_normal((5, dims)).astype(np.float32)
    orc = oracle_mod.FlatIndex("port", dims, m, 16, 64, "l2", capacity=n)
    orc.build(x)
    for ef in (3, 24):
        want = orc.search_many(q, ef, want_counters=True)
        got = run_emu(emu, "l2", coop, x, orc.links(), orc.labels(), q, ef, 2 * m, warps=3, rings=2, grid=2, vh=64, tpr8=True)
        assert got["labels"].tobytes() == want["labels"].tobytes()
        assert got["stats"][:, :3].tolist() == want["counters"][:, :3].tolist()
        for qi in range(q.shape[0]):
            k = int(got["n"][qi])
            assert got["dists"][qi, :k].tobytes() == oracle_mod.dist_many("port", "l2", q[qi], x[got["ids"][qi, :k]]).tobytes()
