"""GPU tests of the error bound the tensor-core scan filter rests on (K6, csrc/scan_umma_kernel.cuh), and of its drop
decisions at numeric and orchestration edges.

The filter drops a (query,row) pair when a lower bound of its distance, built from the TF32 product S under the assumption
|S - q.v| <= rel |q||v|, exceeds the query's k-th exact distance.  A dropped row is never re-scored, so the tripwire of
scan_rescore_kernel cannot see a wrong drop: the bound itself has to be pinned by the product tests here.

a. integer data (exact in TF32, every partial sum an integer below 2^24): the wgmma product equals the float64 product
   exactly, over ragged dims, query / row tile edges, rows past the end of the table, and grids in which every CTA runs
   several tiles (ring parity across tiles, accumulator reset, double-buffered row constants);
b. general data: the product is within fp32-accumulation distance of the product of TF32-cut operands; which cut the
   tensor cores apply (truncation or round-to-nearest-even) is found and printed;
c. worst-case data (every operand loses close to a whole TF32 ulp, all in the same direction): still inside the bound,
   and using more than half of it;
d. pgemb_scan_topk through the filter == the exact kernels == the oracle: near-ties inside the error band with tie-breaks
   across chunks, a sweep of magnitudes, a large common offset, zero rows and a zero query;
e. an assumed bound far too small makes the tripwire fire exactly once per scan, and the result is still the exact one;
f. k at the shared-memory top-k edge and at its maximum, more queries than one query group (both entry points), the
   chunk-policy knobs and the rule that merges a short last chunk into the one before it.

tests/test_capi_emulated.py reuses a, d, e and f on the host-emulated library at small sizes."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_scan_umma import counters, rel_bound, umma_product

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pg():
    import pg_embedding_b200 as pg
    from pg_embedding_b200 import build
    build.build()
    if pg.device_count() < 1:
        pytest.fail("no CUDA device: the product path has no CPU fallback")
    return pg


# ---- operand models -------------------------------------------------------------------------------------------------
MODELS = ("truncate", "rne")


def tf32_cut(x, model):
    """x (float32) cut to TF32's 10 mantissa bits: low 13 bits cleared, or rounded to nearest even."""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    if model == "rne":
        b = b + 0x0FFF + ((b >> 13) & 1)
    return (b & 0xFFFFE000).astype(np.uint32).view(np.float32)


def set_low_bits(x, low):
    """x (float32) with its low 13 mantissa bits replaced by `low`."""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((b & np.uint32(0xFFFFE000)) | np.uint32(low)).view(np.float32)


def model_fits(got, q, x, model):
    """got (nq x nr) within (dim/8 + 16) * 2^-23 * sum|q~_i v~_i| of the float64 product of the cut operands q~, v~
    (the fp32 accumulation of dim products, eight per wgmma k-step, with room to spare)."""
    dims = q.shape[1]
    qt, xt = tf32_cut(q, model).astype(np.float64), tf32_cut(x, model).astype(np.float64)
    tol = (dims / 8 + 16) * 2.0 ** -23 * (np.abs(qt) @ np.abs(xt).T)
    return bool((np.abs(got.astype(np.float64) - qt @ xt.T) <= tol).all())


def worst_case_rows(rng, n, dims, low=0x1FFF, expo=None):
    """All-positive rows, nearly parallel: coordinate i is 2^e_i (1 + u), u < 2^-9, e_i shared by all rows, low 13
    mantissa bits set to `low`.  Truncation then removes close to a whole TF32 ulp (2^-10) from every operand (0x0FFF:
    just under half an ulp, the worst case of rounding), always downwards, so the errors of the dim products add up."""
    e = rng.integers(-3, 4, dims) if expo is None else expo
    return set_low_bits(np.ldexp(1.0 + rng.uniform(0, 2.0 ** -9, (n, dims)), e).astype(np.float32), low)


def _index(pg, metric, x, labels=None):
    idx = pg.HnswIndex(x.shape[1], 4, 8, 16, metric, capacity=max(1, x.shape[0]))
    idx.append(x, labels)
    return idx


# ---- a. exact product on TF32-representable data --------------------------------------------------------------------
INT_SHAPES = [  # dims, rows, nq, r0, nr     (grid = min(tiles, 132): > 396 tiles gives every CTA three or more)
    (1, 300, 1, 1, 299), (4, 1000, 127, 3, 997), (8, 40000, 300, 1, 39999), (31, 700, 128, 5, 695), (32, 513, 129, 1, 512),
    (33, 60001, 129, 1, 60000), (100, 1000, 300, 255, 745), (768, 34100, 300, 1, 34099), (2000, 600, 127, 1, 599),
]


def check_integer_product(pg, shape):
    dims, n, nq, r0, nr = shape
    rng = np.random.default_rng(dims * 7 + nq)
    x = rng.integers(-8, 9, (n, dims)).astype(np.float32)
    q = rng.integers(-8, 9, (nq, dims)).astype(np.float32)
    idx = _index(pg, "l2", x)
    got = umma_product(pg, idx, q, r0, nr)
    idx.close()
    want = q.astype(np.float64) @ x[r0:r0 + nr].astype(np.float64).T
    # equal as values: the sign of a zero sum depends on the zero padding lanes the tensor core adds in
    bad = got != want
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        pytest.fail(f"{int(bad.sum())} of {bad.size} products differ; first at (query, row) {at}: {got[at]} != {want[at]}")


@pytest.mark.parametrize("shape", INT_SHAPES, ids=[f"d{s[0]}n{s[1]}q{s[2]}r{s[3]}" for s in INT_SHAPES])
def test_umma_product_exact_on_integers(pg, shape):
    check_integer_product(pg, shape)


# ---- b. the product against the two operand models ------------------------------------------------------------------
@pytest.fixture(scope="module")
def tf32_model(pg):
    """The operand cut of the tensor cores, from data on which the two models disagree by a whole TF32 ulp per operand:
    all positive, low 13 bits 0x1800 (truncation removes 3/4 ulp, round-to-nearest adds 1/4 ulp)."""
    rng = np.random.default_rng(1)
    x = worst_case_rows(rng, 256, 64, low=0x1800)
    q = worst_case_rows(rng, 16, 64, low=0x1800)
    idx = _index(pg, "l2", x)
    got = umma_product(pg, idx, q, 0, 256)
    idx.close()
    fits = {m: model_fits(got, q, x, m) for m in MODELS}
    print(f"TF32 operand model of the tensor cores: {fits}")
    assert sum(fits.values()) == 1, f"the product fits {'both' if all(fits.values()) else 'neither'} operand model: {fits}"
    return next(m for m in MODELS if fits[m])


MODEL_SHAPES = [  # dims, rows, nq, r0, nr
    (3, 300, 5, 0, 300), (33, 700, 129, 7, 600), (100, 1000, 37, 255, 745), (768, 3000, 130, 1, 2999), (2000, 600, 40, 0, 600),
]


@pytest.mark.parametrize("shape", MODEL_SHAPES, ids=[f"d{s[0]}n{s[1]}q{s[2]}" for s in MODEL_SHAPES])
def test_umma_product_matches_operand_model(pg, tf32_model, shape):
    dims, n, nq, r0, nr = shape
    rng = np.random.default_rng(dims * 13 + n)
    x = rng.standard_normal((n, dims)).astype(np.float32)
    q = rng.standard_normal((nq, dims)).astype(np.float32)
    for f in (2.0 ** 20, 2.0 ** -20, 37.0, 1e-3):      # rows and queries of very different norms
        x[rng.choice(n, n // 10, replace=False)] *= np.float32(f)
    q[0] *= np.float32(2.0 ** -12)
    q[-1] *= np.float32(2.0 ** 12)
    idx = _index(pg, "l2", x)
    got = umma_product(pg, idx, q, r0, nr)
    idx.close()
    fits = {m: model_fits(got, q, x[r0:r0 + nr], m) for m in MODELS}
    print(f"dims={dims}: operand models that fit {fits}")
    assert fits[tf32_model], f"the {tf32_model} model fits the worst-case data but not this product: {fits}"


# ---- c. worst-case data for the bound -------------------------------------------------------------------------------
def check_worst_case_bound(pg, dims, model, n=600, nq=64):
    rng = np.random.default_rng(dims)
    low = 0x1FFF if model == "truncate" else 0x0FFF
    e = rng.integers(-3, 4, dims)
    x, q = worst_case_rows(rng, n, dims, low, e), worst_case_rows(rng, nq, dims, low, e)
    idx = _index(pg, "l2", x)
    got = umma_product(pg, idx, q, 0, n).astype(np.float64)
    idx.close()
    q64, x64 = q.astype(np.float64), x.astype(np.float64)
    bound = rel_bound(dims) / 1.5 * np.outer(np.linalg.norm(q64, axis=1), np.linalg.norm(x64, axis=1))
    ratio = float(np.max(np.abs(got - q64 @ x64.T) / bound))
    print(f"worst-case data, {model} operands, dims={dims}: max err/bound {ratio:.4f}")
    return ratio


@pytest.mark.parametrize("dims", [8, 32, 768, 2000])
def test_umma_product_worst_case_within_bound(pg, tf32_model, dims):
    ratio = check_worst_case_bound(pg, dims, tf32_model)
    assert ratio <= 1.0, f"the TF32 product left the error bound the filter assumes: err/bound {ratio:.4f}"
    # truncation can use 2 * 2^-10 of the bound's 2 * 2^-10 + dim * 2^-21; rounding at most half of that
    floor = 0.5 if tf32_model == "truncate" else 0.2
    assert ratio > floor, f"the data does not stress the bound: err/bound {ratio:.4f}"


# ---- d. drop decisions at the edges ---------------------------------------------------------------------------------
def scan_both_paths(idx, q, k, monkeypatch, what, **env):
    """The exact kernels' result, and the tensor-core path's (with `env` set): equal bytes.  Returns (result, counter deltas)."""
    monkeypatch.setenv("PGEMB_SCAN_TC", "0")
    want = idx.scan_topk(q, k)
    monkeypatch.setenv("PGEMB_SCAN_TC", "2")
    for kk, vv in env.items():
        monkeypatch.setenv(kk, str(vv))
    c0 = counters()
    got = idx.scan_topk(q, k)
    c1 = counters()
    for kk in env:
        monkeypatch.delenv(kk)
    assert got["n"].tobytes() == want["n"].tobytes(), what
    bad = np.argwhere((got["labels"] != want["labels"]) | (got["dists"].view(np.uint32) != want["dists"].view(np.uint32)))
    assert len(bad) == 0, f"{what}: {len(bad)} result slots differ from the exact kernels', first at (query, rank) {tuple(int(i) for i in bad[0])}"
    return got, {key: c1[key] - c0[key] for key in c1}


def assert_no_fallback(dc, what):
    assert dc["tc"] == 1 and dc["fallbacks"] == 0, f"{what}: the tripwire fired (TF32 error bound exceeded): {dc}"


def check_against_oracle(oracle_mod, metric, x, labels, q, got, k, queries):
    """got's rows `queries` == the oracle's distances sorted by (dist, label), the order of the exact path's keys (f2o in
    common.cuh; NaN sorts where the library's NaN bits put it)."""
    n = x.shape[0]
    labels = np.arange(n, dtype=np.uint64) if labels is None else labels
    for i in queries:
        d = np.asarray(oracle_mod.dist_many("port", metric, q[i], x), np.float32).copy()
        gd = got["dists"][i]
        d[np.isnan(d)] = gd[np.isnan(gd)][0] if np.isnan(gd).any() else np.uint32(0x7FFFFFFF).view(np.float32)
        b = d.view(np.uint32)
        key = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000))
        order = np.lexsort((labels, key))[:k]
        assert int(got["n"][i]) == len(order), (metric, i)
        assert got["labels"][i, :len(order)].tolist() == labels[order].tolist(), (metric, i)
        assert got["dists"][i, :len(order)].tobytes() == d[order].tobytes(), (metric, i)


def _sample(nq):
    return sorted({0, nq - 1} | set(range(0, nq, max(1, nq // 6))))


def check_near_ties(pg, oracle_mod, metric, monkeypatch, dims, n, nq=12, k=10):
    """Rows c + r u (u unit, r within 0.1 %) around worst-case-truncation data: every row is inside the error band, so
    the filter keeps all of them and the candidate lists overflow.  Exact duplicates of query 0's k-th neighbour (moved to
    row 0, chunk 0) with smaller labels sit in later chunks: the (dist, label) tie-break crosses chunks."""
    rng = np.random.default_rng(dims + n)
    c = worst_case_rows(rng, 1, dims)[0].astype(np.float64)
    u = rng.standard_normal((n, dims))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    x = set_low_bits(c + 2.0 ** -6 * (1 + 1e-3 * rng.random((n, 1))) * u, 0x1FFF)
    w = rng.standard_normal((nq, dims))
    q = set_low_bits(c + 2.0 ** -8 * w / np.linalg.norm(w, axis=1, keepdims=True), 0x1FFF)
    q[0] = set_low_bits(c, 0x1FFF)
    labels = rng.permutation(n).astype(np.uint64) + np.uint64(10)
    d = np.asarray(oracle_mod.dist_many("port", metric, q[0], x), np.float32)
    kth = int(np.lexsort((labels, d))[k - 1])
    x[[0, kth]] = x[[kth, 0]]
    labels[[0, kth]] = labels[[kth, 0]]
    for lab, at in enumerate((n // 2 + 1, (3 * n) // 4, n - 1)):
        x[at] = x[0]
        labels[at] = np.uint64(lab + 1)
    assert (x > 0).all()
    idx = _index(pg, metric, x, labels)
    got, dc = scan_both_paths(idx, q, k, monkeypatch, f"near ties {metric} dims={dims}")
    idx.close()
    assert_no_fallback(dc, f"near ties {metric} dims={dims}")
    print(f"near ties {metric} dims={dims} n={n}: {dc['rescored'] / max(1, dc['pairs']):.3f} of the pairs re-scored, {dc['overflow']} overflowed lists")
    check_against_oracle(oracle_mod, metric, x, labels, q, got, k, _sample(nq))
    assert 1 in got["labels"][0].tolist(), "the duplicate with the smallest label must displace query 0's k-th neighbour"


def sweep_exponents(metric, x, q, count=9):
    """Exponents e for which x 2^e, q 2^e keep every squared norm and squared distance (L2) or every product of two
    squared norms (cosine: the exact distance divides by sqrt(qn vn)) a normal fp32 with a factor of 4 to spare."""
    x64, q64 = x.astype(np.float64), q.astype(np.float64)
    qn, vn = (q64 ** 2).sum(1), (x64 ** 2).sum(1)
    if metric == "l2":
        d2 = ((q64[:, None, :] - x64[None, :, :]) ** 2).sum(-1)
        small = min(d2[d2 > 0].min(), qn.min(), vn.min())
        lo, hi = np.ceil((-124 - np.log2(small)) / 2), np.floor((126 - np.log2(2 * max(qn.max(), vn.max()))) / 2)
    else:
        lo, hi = np.ceil((-124 - np.log2(qn.min() * vn.min())) / 4), np.floor((126 - np.log2(qn.max() * vn.max())) / 4)
    return sorted({int(e) for e in np.linspace(lo, hi, count).round()} | {0})


def _clustered(rng, n, nq, dims, shift=0.0):
    c = rng.standard_normal((12, dims))
    x = (c[rng.integers(0, 12, n)] + 0.15 * rng.standard_normal((n, dims)) + shift).astype(np.float32)
    q = (c[rng.integers(0, 12, nq)] + 0.15 * rng.standard_normal((nq, dims)) + shift).astype(np.float32)
    return x, q


def check_scale_sweep(pg, oracle_mod, metric, monkeypatch, dims, n, nq=16, k=10):
    """The same clustered data at magnitudes 2^e across the whole range where the norms stay normal fp32: the filter's
    slack must scale with the data (no fallback), and its drops must stay right."""
    rng = np.random.default_rng(40 + dims)
    x, q = _clustered(rng, n, nq, dims, shift=1.0 if metric == "cosine" else 0.0)
    exps = sweep_exponents(metric, x, q)
    print(f"scale sweep {metric} dims={dims}: 2^{exps[0]} .. 2^{exps[-1]}")
    for e in exps:
        xs, qs = np.ldexp(x, e).astype(np.float32), np.ldexp(q, e).astype(np.float32)
        idx = _index(pg, metric, xs)
        got, dc = scan_both_paths(idx, qs, k, monkeypatch, f"{metric} dims={dims} scale 2^{e}")
        idx.close()
        assert_no_fallback(dc, f"{metric} dims={dims} scale 2^{e}")
        check_against_oracle(oracle_mod, metric, xs, None, qs, got, k, _sample(nq)[:3])


def check_offset_and_zeros(pg, oracle_mod, metric, monkeypatch, dims, n, nq=16, k=10):
    """A large common offset (0.01 spread around 100 and 10^4: the whole table is inside the error band, the lists
    overflow); then zero rows and a zero query (cosine: NaN distances, which the filter never drops)."""
    rng = np.random.default_rng(50 + dims)
    for off in (100.0, 1e4):
        x = (off + 0.01 * rng.standard_normal((n, dims))).astype(np.float32)
        q = (off + 0.01 * rng.standard_normal((nq, dims))).astype(np.float32)
        idx = _index(pg, metric, x)
        got, dc = scan_both_paths(idx, q, k, monkeypatch, f"{metric} offset {off}")
        idx.close()
        assert_no_fallback(dc, f"{metric} offset {off}")
        check_against_oracle(oracle_mod, metric, x, None, q, got, k, _sample(nq)[:3])
    x, q = _clustered(rng, n, nq, dims, shift=1.0 if metric == "cosine" else 0.0)
    x[::17] = 0.0
    q[0] = 0.0
    labels = rng.permutation(n).astype(np.uint64)
    idx = _index(pg, metric, x, labels)
    got, dc = scan_both_paths(idx, q, k, monkeypatch, f"{metric} zero vectors")
    idx.close()
    assert_no_fallback(dc, f"{metric} zero vectors")
    check_against_oracle(oracle_mod, metric, x, labels, q, got, k, _sample(nq))


@pytest.mark.parametrize("metric", ["l2", "cosine"])
@pytest.mark.parametrize("dims", [24, 768])
def test_scan_near_ties(pg, oracle_mod, metric, dims, monkeypatch):
    check_near_ties(pg, oracle_mod, metric, monkeypatch, dims, 20000)


@pytest.mark.parametrize("metric", ["l2", "cosine"])
@pytest.mark.parametrize("dims", [24, 128])
def test_scan_scale_sweep(pg, oracle_mod, metric, dims, monkeypatch):
    check_scale_sweep(pg, oracle_mod, metric, monkeypatch, dims, 5000)


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_scan_offset_and_zero_vectors(pg, oracle_mod, metric, monkeypatch):
    check_offset_and_zeros(pg, oracle_mod, metric, monkeypatch, 32, 10000)


# ---- e. the tripwire on the real product ----------------------------------------------------------------------------
def check_tripwire(pg, oracle_mod, metric, monkeypatch, dims, n, nq=16, k=10):
    """PGEMB_SCAN_TC_REL_PPM=1 assumes an error bound of 1e-6 |q||v|; the worst-case data's product misses by ~2^-9, so
    the first chunk's re-scoring sees it: one fallback, and the exact kernels' result."""
    rng = np.random.default_rng(60 + dims)
    e = rng.integers(-3, 4, dims)
    x, q = worst_case_rows(rng, n, dims, 0x1FFF, e), worst_case_rows(rng, nq, dims, 0x1FFF, e)
    idx = _index(pg, metric, x)
    got, dc = scan_both_paths(idx, q, k, monkeypatch, f"tripwire {metric}", PGEMB_SCAN_TC_REL_PPM=1)
    print(f"tripwire {metric} dims={dims}: {dc['fallbacks']} fallback(s)")
    assert dc["tc"] == 1 and dc["fallbacks"] == 1 and dc["exact"] == 1, dc
    _, dc = scan_both_paths(idx, q, k, monkeypatch, f"default bound {metric}")
    assert_no_fallback(dc, f"default bound {metric}")
    idx.close()
    check_against_oracle(oracle_mod, metric, x, None, q, got, k, _sample(nq)[:3])


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_scan_tripwire_fires_once(pg, oracle_mod, metric, monkeypatch):
    check_tripwire(pg, oracle_mod, metric, monkeypatch, 256, 3000)


# ---- f. orchestration edges -----------------------------------------------------------------------------------------
def check_k_edges(pg, oracle_mod, metric, monkeypatch, ks, n, dims=16, nq=24):
    """k at the edge of the re-scoring kernel's shared-memory top-k (256 / 257) and at the maximum (4096: a first chunk of
    8192 rows, the top-k in global memory)."""
    rng = np.random.default_rng(70)
    x, q = _clustered(rng, n, nq, dims, shift=1.0 if metric == "cosine" else 0.0)
    labels = rng.permutation(n).astype(np.uint64) + np.uint64(1)
    idx = _index(pg, metric, x, labels)
    for k in ks:
        got, dc = scan_both_paths(idx, q, k, monkeypatch, f"{metric} k={k}")
        assert_no_fallback(dc, f"{metric} k={k}")
        check_against_oracle(oracle_mod, metric, x, labels, q, got, k, _sample(nq)[:3])
    idx.close()


def scan_device(idx, q, k):
    """pgemb_scan_topk_device: device pointers on a real device, host memory on the emulated library."""
    from pg_embedding_b200 import _lib
    import torch
    lib = _lib.load()
    nq = q.shape[0]
    ol, od, on = np.zeros((nq, k), np.uint64), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32)
    if torch.cuda.is_available():
        tq, tl, td, tn = (torch.from_numpy(a).cuda() for a in (q, ol.view(np.int64), od, on))
        _lib.check(lib.pgemb_scan_topk_device(idx.dev, nq, tq.data_ptr(), k, tl.data_ptr(), td.data_ptr(), tn.data_ptr(), None))
        torch.cuda.synchronize()
        return {"labels": tl.cpu().numpy().view(np.uint64), "dists": td.cpu().numpy(), "n": tn.cpu().numpy()}
    _lib.check(lib.pgemb_scan_topk_device(idx.dev, nq, q.ctypes.data_as(C.c_void_p), k, ol.ctypes.data_as(C.c_void_p), od.ctypes.data_as(C.c_void_p),
                                          on.ctypes.data_as(C.c_void_p), None))
    return {"labels": ol, "dists": od, "n": on}


def check_query_groups(pg, oracle_mod, metric, monkeypatch, n, nq=4096 + 37, dims=32, k=10):
    """More queries than one group of the tensor-core path (4096): two groups, both entry points, queries on both sides
    of the split against the oracle."""
    rng = np.random.default_rng(80)
    x, q = _clustered(rng, n, nq, dims, shift=1.0 if metric == "cosine" else 0.0)
    idx = _index(pg, metric, x)
    got, dc = scan_both_paths(idx, q, k, monkeypatch, f"{metric} nq={nq}")
    assert dc["tc"] == (nq + 4095) // 4096 and dc["fallbacks"] == 0, dc
    monkeypatch.setenv("PGEMB_SCAN_TC", "2")
    dev = scan_device(idx, q, k)
    idx.close()
    for key in ("labels", "dists", "n"):
        assert dev[key].tobytes() == got[key].tobytes(), key
    check_against_oracle(oracle_mod, metric, x, None, q, got, k, [0, 4095, 4096, nq - 1])


def check_chunk_policy(pg, oracle_mod, metric, monkeypatch, n, dims=16, nq=20, k=10):
    """The chunk-policy knobs.  With n = 10772 (GPU) or 1044 (emulator) both settings end in the "no sliver" merge:
    growth 3 gives chunks 256, 768, 2304 and then 7412 = 6912 + the 500 rows left over (1044: 256 + 788); chunks capped
    at 256 rows end in 256 + 20."""
    rng = np.random.default_rng(90)
    x, q = _clustered(rng, n, nq, dims, shift=1.0 if metric == "cosine" else 0.0)
    labels = rng.permutation(n).astype(np.uint64) + np.uint64(5)
    idx = _index(pg, metric, x, labels)
    for env in ({"PGEMB_SCAN_TC_CHUNK_MAX_LOG2": 8}, {"PGEMB_SCAN_TC_GROWTH": 3}, {"PGEMB_SCAN_TC_CHUNK_MAX_LOG2": 8, "PGEMB_SCAN_TC_GROWTH": 3}):
        got, dc = scan_both_paths(idx, q, k, monkeypatch, f"{metric} {env}", **env)
        assert_no_fallback(dc, f"{metric} {env}")
        check_against_oracle(oracle_mod, metric, x, labels, q, got, k, _sample(nq)[:3])
    idx.close()


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_scan_k_edges(pg, oracle_mod, metric, monkeypatch):
    check_k_edges(pg, oracle_mod, metric, monkeypatch, (256, 257, 4096), 30000)


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_scan_query_groups(pg, oracle_mod, metric, monkeypatch):
    check_query_groups(pg, oracle_mod, metric, monkeypatch, 5000)


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_scan_chunk_policy(pg, oracle_mod, metric, monkeypatch):
    check_chunk_policy(pg, oracle_mod, metric, monkeypatch, 10772)
