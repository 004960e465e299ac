"""Every device distance path against hnsw_dist_func, bit for bit, at each kernel's loop and tail boundaries.

The reference's distances come out of distfunc.c as vectorised by `gcc -Ofast` (DESIGN.md section 4); dist_exact.cuh
restates that summation order, and every kernel that scores a pair restates it again with its own main loop, unrolling
and tail: dist_pairs_kernel / dist_gather_kernel (distance_exact), the traversal's score_row4 / score_row8_l2 (query
transposed in shared memory, rows through the rings, in throughput and latency mode), the exact scan (scan_dist_kernel,
scan_tile_kernel, the tensor-core path's re-scoring) and the binds (node_dist, heuristic_block_staged).  An ordering
slip in any of them shows only at the dimensions whose residues reach the slipped branch, so DIMS below is derived from
those loops, and the data is drawn so that a plausible wrong order gives other bits (the discrimination guard proves
that on the very pairs the kernels are checked on).

tests/test_capi_emulated.py runs the same check_* bodies on the emulated library with EMU_DIMS."""
import ctypes as C
import json
import os
import re
import tempfile

import numpy as np
import pytest

from test_gpu_parity import checkers, kernel_mode

pytestmark = pytest.mark.gpu

METRICS = ["l2", "cosine", "manhattan"]

# L2 (dist_exact.cuh, search_kernel.cuh): 16-float blocks, nb = dim // 16, tail r = dim % 16 through l2_tail_exact
# (r 1-3: scalars only; 4-7: the 4-wide block; 8: the 8-wide block alone; 9-11: 8-wide + scalars; 12-15: 8 + 4 + scalars).
# score_row4 takes the blocks in pairs (npair = nb // 2) and then an odd block; score_row8_l2 in fours (nquad = nb // 4)
# and then nb % 4 single blocks.  Cosine / manhattan: 4-float steps, n4 = dim // 4, tail dim % 4; score_row4 runs
# pipelined groups of 8 steps (nit = n4 // 8), then n4 % 8 single steps.  scan_tile_kernel stages 64-dimension chunks
# of the main part, the last one partial, and reads the tail from global memory.  The traversal stages the query in
# strides of 256 floats.
DIMS = sorted(set(
    # every L2 residue with nb = 0, 1, 2 (no block; score_row4's lone odd block; its first full pair); every dim % 4
    # tail with n4 = 0..12 (nit = 0 with 0-7 single steps, nit = 1 with 0-4 single steps)
    list(range(1, 49))
    # score_row4 L2 nb = 3 (one pair + odd block): r = 5 / 11; cosine n4 = 13 / 14 (nit = 1 + 5 / 6 steps)
    + [53, 59]
    # scan tile chunks: main part of 48 (cosine 60) in one partial chunk, exactly one chunk of 64 (L2 nb = 4: two pairs,
    # nquad = 1; cosine nit = 2 exactly), one chunk + tail 1, one chunk + tail 15 (cosine: 64 + a partial chunk of 12)
    + [63, 64, 65, 79]
    # cosine n4 = 17 (nit = 2 + one step) with tail 3; L2 nb = 4, r = 7
    + [71]
    # L2 nb = 5 (npair = 2 + odd block; nquad = 1 + one block): r = 6 (4-wide block + 2 scalars), r = 12
    + [86, 92]
    # L2 nb = 7 (npair = 3 + odd block; nquad = 1 + three blocks): r = 6, 12, 15 (127: scan chunk 64 + partial 48)
    + [118, 124, 127]
    # L2 nb = 8 (nquad = 2, no remainder): r = 0, r = 9 (8-wide block + 1 scalar); 129: scan two full chunks + tail 1
    + [128, 129, 137]
    # L2 nb = 9 (nquad = 2 + one block): r = 6, 14
    + [150, 158]
    # query staging stride of 256: one float short, exact, one over; the second stride
    + [255, 256, 257, 511, 513]
    # BASELINE row shapes and their neighbours (1551: nb = 96, r = 15)
    + [767, 768, 769, 1535, 1536, 1537, 1551]
    # rows of >= 4096 bytes take 8 lanes per row by default: the tails that go through l2_tail_exact's 8-wide block there
    + [1030, 1033, 1036, 1038]
    # the largest dims a page holds
    + [1999, 2000]
))

# binds (node_dist, the staged heuristic, the stored-node query of the insert's search): every residue class, then
# one dim per boundary group above
INSERT_DIMS = list(range(1, 17)) + [17, 24, 28, 39, 53, 79, 86, 127, 137, 150, 257, 513, 769, 1038, 1551, 2000]

# the emulated leg: every residue with 0-2 L2 blocks and a few boundary dims of each path
EMU_DIMS = list(range(1, 49)) + [53, 71, 86, 127, 137, 257]
EMU_INSERT_DIMS = [3, 5, 6, 8, 9, 12, 14, 15, 39, 86]      # with 80 rows

N_ROWS, N_QUERIES = 150, 12          # 150 rows: a partial 64-row scan tile, ragged 32-row / 8-row hop groups
COSINE_OFFSET = 4.0


@pytest.fixture(scope="module")
def pg():
    import pg_embedding_b200 as pg
    from pg_embedding_b200 import build
    build.build()
    if pg.device_count() < 1:
        pytest.fail("no CUDA device: the product path has no CPU fallback")
    return pg


# ---------------------------------------------------------------------------------------------------
# data that tells summation orders apart
# ---------------------------------------------------------------------------------------------------
def make_case(metric, dim, n=N_ROWS, nq=N_QUERIES):
    """Rows and queries whose coordinates are +-(1+u) 2^e, e uniform in [-8, 8]: a sum mixes terms of very different
    size, so where it rounds depends on the order it adds them in.  Queries 0-1 are exact copies of stored rows (L2 0,
    cosine a few ulps around 0, possibly negative), 2-4 near copies (the L2 differences nearly cancel), 5 a scaled copy
    (cosine ~0); two rows are duplicates of others.  Cosine adds a common offset.  No zero vector and no sum or norm
    product near the fp32 range: NaN and overflow are outside the parity claim."""
    rng = np.random.default_rng(7919 * dim + METRICS.index(metric))

    def coords(shape):
        e = rng.integers(-8, 9, size=shape)
        return (rng.choice([-1.0, 1.0], size=shape) * (1.0 + rng.random(shape)) * np.exp2(e)).astype(np.float32)

    x = coords((n, dim))
    if metric == "cosine":
        x += np.float32(COSINE_OFFSET)
    x[n - 1], x[n - 2] = x[0], x[1]
    q = coords((nq, dim))
    if metric == "cosine":
        q += np.float32(COSINE_OFFSET)
    src = rng.choice(n - 2, 6, replace=False)
    q[0:2] = x[src[0:2]]
    for i, frac, scale in ((2, 1.0, -12), (3, 0.5, -16), (4, 0.125, -20)):   # share of coordinates moved, by how much
        move = rng.random(dim) < frac
        move[rng.integers(dim)] = True
        wiggle = (1.0 + np.exp2(scale) * rng.standard_normal(dim)).astype(np.float32)
        q[i] = np.where(move, x[src[i]] * wiggle, x[src[i]])
    q[5] = x[src[5]] * np.float32(2.0)
    labels = (np.arange(n, dtype=np.uint64)[::-1] << np.uint64(20)) | np.uint64(3)     # labels order differently from ids
    return np.ascontiguousarray(x), np.ascontiguousarray(q), labels


def oracle_dists(oracle_mod, metric, x, q):
    """{checker: float32[nq, n]}: one hnsw_dist_func call per (query, row) pair."""
    nq, n = q.shape[0], x.shape[0]
    a, b = np.repeat(q, n, axis=0), np.tile(x, (nq, 1))
    return {w: oracle_mod.dist_many(w, metric, a, b).reshape(nq, n) for w in checkers(oracle_mod)}


# ---------------------------------------------------------------------------------------------------
# discrimination guard: plausible wrong orders, restated in numpy, must disagree with the oracle on these pairs
# ---------------------------------------------------------------------------------------------------
def _hsum4(add, s, swap):
    # the reference: (s0 + s2) + (s1 + s3); swap: (s0 + s1) + (s2 + s3)
    return add(add(s[0], s[1]), add(s[2], s[3])) if swap else add(add(s[0], s[2]), add(s[1], s[3]))


def _sum_l2_blocks(t, dim, add, zero, swap=False, tail_first=False):
    """distfunc.c's AVX2 loop as compiled: 8 lanes over 16-float blocks, horizontal sum, the vectorised tail."""
    main = dim & ~15
    S = [zero] * 8
    for i in range(0, main, 16):
        for j in range(8):
            S[j] = add(S[j], add(t(i + j), t(i + 8 + j)))
    if tail_first:
        for k in range(main, dim):
            S[0] = add(S[0], t(k))
        main = dim
    res = _hsum4(add, [add(S[j], S[j + 4]) for j in range(4)], swap)
    pos, r = main, dim - main
    u = [zero] * 4
    if r >= 8:
        u = [add(t(pos + j), t(pos + 4 + j)) for j in range(4)]
        pos, r = pos + 8, r - 8
        if r < 4:
            res = add(res, _hsum4(add, u, swap))
    if r >= 4:
        res = add(res, _hsum4(add, [add(t(pos + j), u[j]) for j in range(4)], swap))
        pos, r = pos + 4, r - 4
    for k in range(pos, pos + r):
        res = add(res, t(k))
    return res


def _sum_4lanes(t, dim, add, zero, swap=False, tail_first=False):
    """distfunc.c's cosine / manhattan loops as compiled: 4 lanes, horizontal sum, scalar tail."""
    main = dim & ~3
    s = [zero] * 4
    for i in range(0, main, 4):
        for j in range(4):
            s[j] = add(s[j], t(i + j))
    if tail_first:
        for k in range(main, dim):
            s[0] = add(s[0], t(k))
        main = dim
    res = _hsum4(add, s, swap)
    for k in range(main, dim):
        res = add(res, t(k))
    return res


def _sum_sequential(t, dim, add, zero):
    res = zero
    for k in range(dim):
        res = add(res, t(k))
    return res


def _orders(metric):
    """name -> sum(t, dim, add, zero): the reference's order first, then the wrong ones."""
    ref, other = (_sum_l2_blocks, _sum_4lanes) if metric == "l2" else (_sum_4lanes, _sum_l2_blocks)
    return {
        "reference": ref,
        "sequential": _sum_sequential,
        "other lane count": other,      # L2 on 4 lanes; cosine / manhattan on L2's 8 lanes of 16-float blocks
        "tail before the horizontal sum": lambda t, dim, add, zero: ref(t, dim, add, zero, tail_first=True),
        "(s0+s1)+(s2+s3)": lambda t, dim, add, zero: ref(t, dim, add, zero, swap=True),
    }


def restated_dists(metric, a, b, order):
    """float32[pairs] in the given order, fp32 arithmetic rounded at every step (numpy never contracts to FMA)."""
    f = np.float32
    if order == "float64":
        a64, b64 = a.astype(np.float64), b.astype(np.float64)
        if metric == "l2":
            return np.sqrt(((a64 - b64) ** 2).sum(1)).astype(f)
        if metric == "manhattan":
            return np.abs(a64 - b64).sum(1).astype(f)
        return (1.0 - (a64 * b64).sum(1) / np.sqrt((a64 * a64).sum(1) * (b64 * b64).sum(1))).astype(f)
    red = _orders(metric)[order]
    dim, zero = a.shape[1], np.zeros(a.shape[0], f)

    def total(terms):
        return red(lambda k: terms[:, k], dim, np.add, zero)
    if metric == "l2":
        d = a - b
        return np.sqrt(total(d * d))
    if metric == "manhattan":
        return total(np.abs(a - b))
    dot, na, nb = total(b * a), total(a * a), total(b * b)
    return (1.0 - dot.astype(np.float64) / np.sqrt((nb * na).astype(np.float64))).astype(f)


def order_can_differ(metric, dim, order):
    """Whether `order` is a different rounding sequence from the reference's at this dim.  The sums are rebuilt
    symbolically with hash-consed nodes (fp addition is commutative, and 0 + t == t for the nonzero terms here); two
    orders round alike for every input exactly when their trees coincide.  The float64 order rounds once where the
    reference rounds each term and partial sum: a different result is possible from two terms on."""
    if order == "float64":
        return dim >= 2
    nodes = {}

    def add(p, q):
        if p == -1:
            return q
        if q == -1:
            return p
        return nodes.setdefault((min(p, q), max(p, q)), dim + len(nodes))
    orders = _orders(metric)
    return orders[order](lambda k: k, dim, add, -1) != orders["reference"](lambda k: k, dim, add, -1)


WRONG_ORDERS = ["sequential", "float64", "other lane count", "tail before the horizontal sum", "(s0+s1)+(s2+s3)"]


def check_discrimination(oracle_mod, metric, dims):
    """The numpy restatement of the reference's order equals the oracle on every pair; each wrong order that can give
    other bits at a dim does so on at least one of that dim's pairs.  Without the second half 'bits equal' below would
    prove little: inputs on which every order agrees cannot catch a kernel that sums in the wrong one."""
    exempt = []
    for dim in dims:
        x, q, _ = make_case(metric, dim)
        want = oracle_dists(oracle_mod, metric, x, q)
        a, b = np.repeat(q, x.shape[0], axis=0), np.tile(x, (q.shape[0], 1))
        ref = restated_dists(metric, a, b, "reference")
        for w, d in want.items():
            assert ref.tobytes() == d.ravel().tobytes(), (metric, dim, w, "the numpy restatement is wrong")
        for order in WRONG_ORDERS:
            if not order_can_differ(metric, dim, order):
                exempt.append((dim, order))
                continue
            got = restated_dists(metric, a, b, order)
            assert got.tobytes() != ref.tobytes(), (metric, dim, order, "the data cannot tell this order from the reference's")
    # exempt: dims below one 16-float block, and the tail's place where there is no tail
    block = 16 if metric == "l2" else 4
    assert all(d < 16 or (o == "tail before the horizontal sum" and d % block == 0) for d, o in exempt), (metric, exempt)
    return exempt


@pytest.mark.parametrize("metric", METRICS)
def test_discrimination_guard(oracle_mod, metric):
    check_discrimination(oracle_mod, metric, DIMS)


# ---------------------------------------------------------------------------------------------------
# the stand-alone distance entry points
# ---------------------------------------------------------------------------------------------------
def check_dist_entry_points(pg, oracle_mod, metric, dims):
    """pgemb_dist_batch on every (query, row) pair and with a broadcast query; pgemb_dist_gather (queries at `dim`
    stride, rows at the index's padded stride, cached norms) in a shuffled order, and NaN for ids at or beyond the
    index's size -- also for those below its capacity."""
    for dim in dims:
        x, q, labels = make_case(metric, dim)
        nq, n = q.shape[0], x.shape[0]
        want = oracle_dists(oracle_mod, metric, x, q)
        got = pg.dist_batch(metric, np.repeat(q, n, axis=0), np.tile(x, (nq, 1))).reshape(nq, n)
        for w, d in want.items():
            assert got.tobytes() == d.tobytes(), (metric, dim, w, np.argwhere(got != d)[:4])
        for i in (0, 2, 5, nq - 1):
            assert pg.dist_batch(metric, q[i], x).tobytes() == want["port"][i].tobytes(), (metric, dim, "broadcast", i)
        idx = pg.HnswIndex(dim, 4, 8, 16, metric, capacity=n + 8)     # ids in [n, n + 8): allocated rows never written
        idx.append(x, labels)
        rng = np.random.default_rng(dim)
        ids = np.stack([rng.permutation(n) for _ in range(nq)]).astype(np.uint32)
        got = idx.dist_gather(q, ids)
        for w, d in want.items():
            assert got.tobytes() == np.take_along_axis(d, ids.astype(np.int64), 1).tobytes(), (metric, dim, w, "gather")
        bad = ids.copy()
        bad[:, ::5] = np.uint32(n) + bad[:, ::5] % 8           # beyond the index's size, inside its capacity
        bad[:, 3] = np.uint32(n + 8)                            # the first id beyond the capacity
        bad[:, 4] = np.uint32(0xFFFFFFFF)
        out = idx.dist_gather(q, bad)
        oob = bad >= n
        assert np.isnan(out[oob]).all(), (metric, dim)
        assert out[~oob].tobytes() == np.take_along_axis(want["port"], ids.astype(np.int64), 1)[~oob].tobytes()
        idx.close()


@pytest.mark.parametrize("metric", METRICS)
def test_dist_entry_points(pg, oracle_mod, metric):
    check_dist_entry_points(pg, oracle_mod, metric, DIMS)


# ---------------------------------------------------------------------------------------------------
# the traversal: every node scored and returned (ef = n)
# ---------------------------------------------------------------------------------------------------
_SEARCH_ENV = ("PGEMB_COOP_WARPS", "PGEMB_L2_TPR8", "PGEMB_L2_TPR8_MIN_BYTES", "PGEMB_RES_GLOBAL")


def traversal_modes(metric):
    """(name, PGEMB_COOP, other settings, the kernel it must launch: (latency mode, lanes per row, results in global
    memory), warps per CTA: "several" / "one" / None for any).  L2 pins its lanes per row: the default takes 8 for rows of
    >= 4 KB.  Latency mode gives every row group of a hop its own warp; the one-warp variant leaves the owner warp alone."""
    four = {"PGEMB_L2_TPR8": "0"} if metric == "l2" else {}
    eight = {"PGEMB_L2_TPR8": "1", "PGEMB_L2_TPR8_MIN_BYTES": "0"}
    modes = [("latency", "1", dict(four), (True, 4, False), "several"),
             ("latency, one warp", "1", dict(four, PGEMB_COOP_WARPS="1"), (True, 4, False), "one"),
             ("throughput", "0", dict(four), (False, 4, False), None),
             ("results in global memory", "0", {"PGEMB_RES_GLOBAL": "1"}, (False, 4, True), None)]
    if metric == "l2":
        modes += [("latency, 8 lanes", "1", eight, (True, 8, False), "several"),
                  ("latency, 8 lanes, one warp", "1", dict(eight, PGEMB_COOP_WARPS="1"), (True, 8, False), "one"),
                  ("throughput, 8 lanes", "0", eight, (False, 8, False), None)]
    return modes


def traversal_launches(run):
    """Runs `run()` and returns [(kernel template arguments or None, threads per CTA)] of the traversal launches it made.
    On a device they come from torch.profiler's CUDA activity trace: search_kernel<METRIC, COOP, TPR, RESG> and the block
    size.  On the emulated library its runtime's launch log gives the block size of every launch with dynamic shared
    memory (only the traversal kernel has some here), without the kernel's name."""
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
            if e.get("cat") == "kernel" and "search_kernel" in e.get("name", ""):
                m = re.search(r"search_kernel<\s*(\d+),\s*(true|false),\s*(\d+),\s*(true|false)\s*>", e["name"])
                assert m, e["name"]
                out.append(((int(m[1]), m[2] == "true", int(m[3]), m[4] == "true"), int(e["args"]["block"][0])))
        return out
    from pg_embedding_b200 import _lib
    lib = _lib.load()
    cap = 4096
    threads, smem = (C.c_uint * cap)(), (C.c_size_t * cap)()
    lib.emu_launch_log.argtypes = [C.POINTER(C.c_uint), C.POINTER(C.c_size_t), C.c_int]
    lib.emu_launch_log(threads, smem, cap)               # forget what came before
    run()
    k = lib.emu_launch_log(threads, smem, cap)
    assert k <= cap
    return [(None, int(threads[i])) for i in range(k) if smem[i] > 0]


RING_STEPS = (1, -1, 2, -2, 5, -5, 11, -11, 23, -23, 37, -37, 61, -61, 70, -70)   # maxM = 16 distinct neighbours for n = 150


def ring_graph(n, m=8):
    """Link lists in which every node is reachable from every other: node i links to i + s (mod n) for s in RING_STEPS.
    With ef = n a search then scores and returns every node (a graph the heuristic built would leave some unreached).
    A hop of 16 neighbours is two row groups of 8 at 4 lanes per row and four of 4 at 8 lanes, so latency mode runs
    more than one warp."""
    assert 2 * m == len(RING_STEPS)
    links = np.zeros((n, 2 * m + 1), np.uint32)
    links[:, 0] = 2 * m
    for c, st in enumerate(RING_STEPS):
        links[:, 1 + c] = (np.arange(n) + st) % n
    return links


def check_traversal(pg, oracle_mod, metric, dims, monkeypatch, latency_queries=N_QUERIES):
    """ef = n on a graph where every node is reachable: every node is scored and returned.  Labels, counts and traversal
    counters equal the oracle's search on the same graph; every returned distance equals hnsw_dist_func's bits.  Latency
    mode runs the first `latency_queries` queries, at most two per launch, so that it is chosen on any device (it needs
    no more queries than SMs).  At the smallest and the largest dim each mode's launches are observed: the kernel each
    setting names (on a device) and the warps per CTA, so that no two modes quietly become the same kernel."""
    for dim in dims:
        x, q, labels = make_case(metric, dim)
        n, m = x.shape[0], 8
        want = oracle_dists(oracle_mod, metric, x, q)
        links = ring_graph(n, m)
        orc = oracle_mod.FlatIndex("port", dim, m, 32, n, metric, capacity=n)
        orc.load_graph(x, links, labels)
        ws = orc.search_many(q, n, want_counters=True)
        assert ws["n"].tolist() == [n] * q.shape[0]
        idx = pg.HnswIndex(dim, m, 32, n, metric, capacity=n)
        idx.append(x, labels, links)
        for name, coop, env, kernel, warps in traversal_modes(metric):
            nq = latency_queries if coop == "1" else q.shape[0]
            step = 2 if coop == "1" else nq
            outs = []

            def run():
                outs.extend(idx.search_batch(q[i:min(i + step, nq)], n, want_stats=True) for i in range(0, nq, step))
            with kernel_mode(coop), monkeypatch.context() as mp:
                for k in _SEARCH_ENV:
                    mp.delenv(k, raising=False)
                for k, v in env.items():
                    mp.setenv(k, v)
                if dim in (dims[0], dims[-1]):
                    launches = traversal_launches(run)
                    assert len(launches) == len(range(0, nq, step)), (metric, dim, name, launches)
                    for args, threads in launches:
                        assert args is None or args == (METRICS.index(metric),) + kernel, (metric, dim, name, args)
                        assert warps is None or (threads == 32) == (warps == "one"), (metric, dim, name, threads)
                else:
                    run()
            out = {key: np.concatenate([o[key] for o in outs]) for key in ("n", "labels", "ids", "dists", "stats")}
            assert out["n"].tolist() == ws["n"][:nq].tolist(), (metric, dim, name)
            assert out["labels"].tobytes() == ws["labels"][:nq].tobytes(), (metric, dim, name)
            assert out["stats"][:, :3].tolist() == ws["counters"][:nq, :3].tolist(), (metric, dim, name)
            for i in range(nq):
                ids = out["ids"][i].astype(np.int64)
                for w, d in want.items():
                    assert out["dists"][i].tobytes() == d[i, ids].tobytes(), \
                        (metric, dim, name, w, i, np.flatnonzero(out["dists"][i] != d[i, ids])[:4])
        idx.close()
        orc.close()


@pytest.mark.parametrize("metric", METRICS)
def test_traversal_distances(pg, oracle_mod, metric, monkeypatch):
    check_traversal(pg, oracle_mod, metric, DIMS, monkeypatch)


# ---------------------------------------------------------------------------------------------------
# the exact scan: k = n returns every row's distance
# ---------------------------------------------------------------------------------------------------
def scan_modes(metric):
    modes = [("per pair", {"PGEMB_SCAN_TILED": "0", "PGEMB_SCAN_TC": "0"}),
             ("tiled", {"PGEMB_SCAN_TILED": "1", "PGEMB_SCAN_TC": "0"})]
    if metric != "manhattan":
        modes.append(("tensor-core filter, exact re-scoring", {"PGEMB_SCAN_TC": "2"}))
    return modes


def scan_device(idx, q, k):
    """pgemb_scan_topk_device, called as check_device_scan_edge_cases calls it (host memory on the emulated library)."""
    import torch
    from pg_embedding_b200 import _lib
    lib = _lib.load()
    nq = q.shape[0]
    ol = np.zeros((nq, k), np.uint64); od = np.zeros((nq, k), np.float32); on = np.zeros(nq, np.int32)
    if torch.cuda.is_available():
        tq = torch.from_numpy(q).cuda(); tl = torch.from_numpy(ol.view(np.int64)).cuda(); td = torch.from_numpy(od).cuda(); tn = torch.from_numpy(on).cuda()
        _lib.check(lib.pgemb_scan_topk_device(idx.dev, nq, tq.data_ptr(), k, tl.data_ptr(), td.data_ptr(), tn.data_ptr(), None))
        torch.cuda.synchronize()
        return {"labels": tl.cpu().numpy().view(np.uint64), "dists": td.cpu().numpy(), "n": tn.cpu().numpy()}
    _lib.check(lib.pgemb_scan_topk_device(idx.dev, nq, q.ctypes.data_as(C.c_void_p), k, ol.ctypes.data_as(C.c_void_p),
                                          od.ctypes.data_as(C.c_void_p), on.ctypes.data_as(C.c_void_p), None))
    return {"labels": ol, "dists": od, "n": on}


def check_scan(pg, oracle_mod, metric, dims, monkeypatch):
    """pgemb_scan_topk and pgemb_scan_topk_device with k = n under each kernel path: every row's distance bits, in
    ascending (dist, label) order, the same bytes from both entry points."""
    from test_gpu_scan_umma import counters
    for dim in dims:
        x, q, labels = make_case(metric, dim)
        n = x.shape[0]
        want = oracle_dists(oracle_mod, metric, x, q)
        idx = pg.HnswIndex(dim, 4, 8, 16, metric, capacity=n)
        idx.append(x, labels)
        for name, env in scan_modes(metric):
            with monkeypatch.context() as mp:
                for k in ("PGEMB_SCAN_TILED", "PGEMB_SCAN_TC"):
                    mp.delenv(k, raising=False)
                for k, v in env.items():
                    mp.setenv(k, v)
                c0 = counters()
                host = idx.scan_topk(q, n)
                c1 = counters()
                dev = scan_device(idx, q, n)
            if "PGEMB_SCAN_TC" in env and env["PGEMB_SCAN_TC"] == "2":
                assert c1["tc"] == c0["tc"] + 1 and c1["fallbacks"] == c0["fallbacks"], (metric, dim, name, "not the tensor-core path")
            else:
                assert c1["exact"] == c0["exact"] + 1 and c1["tc"] == c0["tc"], (metric, dim, name)
            for key in ("labels", "dists", "n"):
                assert dev[key].tobytes() == host[key].tobytes(), (metric, dim, name, key)
            assert host["n"].tolist() == [n] * q.shape[0]
            for w, d in want.items():
                for i in range(q.shape[0]):
                    order = sorted(zip(d[i].tolist(), labels.tolist()))
                    assert host["labels"][i].tolist() == [o[1] for o in order], (metric, dim, name, w, i)
                    assert host["dists"][i].tobytes() == np.array([o[0] for o in order], np.float32).tobytes(), (metric, dim, name, w, i)
        idx.close()


@pytest.mark.parametrize("metric", METRICS)
def test_scan_distances(pg, oracle_mod, metric, monkeypatch):
    check_scan(pg, oracle_mod, metric, DIMS, monkeypatch)


# ---------------------------------------------------------------------------------------------------
# binds: distances between stored rows decide the link lists
# ---------------------------------------------------------------------------------------------------
def check_insert(pg, oracle_mod, metric, dims, monkeypatch, n=N_ROWS):
    """insert_many, one hnsw_bind_point, insert_many again, with m = 2 or 3 so lists fill and back-links are re-pruned;
    the heuristic with its rows staged in shared memory (the default for single binds) and without.  The link lists equal
    the sequential build's byte for byte: the bind distances (node_dist, the staged rows, the insert's search from a
    stored node) cannot be observed otherwise."""
    for dim in dims:
        x, _, _ = make_case(metric, dim, n=n)
        m, efc = 2 + dim % 2, 16
        wants = {}
        for w in checkers(oracle_mod):
            orc = oracle_mod.FlatIndex(w, dim, m, efc, 16, metric, capacity=n)
            orc.build(x)
            wants[w] = orc.links()
            orc.close()
        for staged in ("1", "0"):
            with monkeypatch.context() as mp:
                mp.setenv("PGEMB_SELECT_STAGED", staged)
                idx = pg.HnswIndex(dim, m, efc, 16, metric, capacity=n)
                idx.insert_many(x[:n // 2])
                idx.insert(x[n // 2])
                idx.insert_many(x[n // 2 + 1:])
                got = idx.links()
                idx.close()
            for w, want in wants.items():
                bad = np.flatnonzero((got != want).any(1))
                assert bad.size == 0, (metric, dim, staged, w, bad[:8])


@pytest.mark.parametrize("metric", METRICS)
def test_insert_links(pg, oracle_mod, metric, monkeypatch):
    check_insert(pg, oracle_mod, metric, INSERT_DIMS, monkeypatch)
