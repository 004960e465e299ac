"""Pins the C restatement (oracle/hnsw_oracle.c, `port`) to the UNMODIFIED compiled reference bit for bit: distances for
every dim / metric, link lists after sequential builds, and search results -- including duplicate vectors (exact distance
ties).  The reference's outputs for these seeded inputs are recorded in tests/golden/ref_compare.json (the leading 64 bits of
the SHA-256 of the raw bytes, written by tests/golden/gen_ref_fixtures.py from oracle/_ref), so the comparison needs no reference tree."""
import hashlib
import json
import os

import numpy as np
import pytest

METRICS = ["l2", "cosine", "manhattan"]
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "ref_compare.json")))


def digest(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def distance_outputs(oracle_mod, which, metric):
    rng = np.random.default_rng(7)
    dims = list(range(1, 70)) + [96, 100, 127, 128, 129, 255, 256, 300, 768, 769, 1000, 1536, 2000]
    pairs, broadcast = [], []
    for dim in dims:
        a = rng.standard_normal((64, dim)).astype(np.float32)
        b = rng.standard_normal((64, dim)).astype(np.float32)
        # mix magnitudes so that rounding order matters
        a *= rng.choice([1e-3, 1.0, 37.0], size=(64, 1)).astype(np.float32)
        pairs.append(oracle_mod.dist_many(which, metric, a, b))
        broadcast.append(oracle_mod.dist_many(which, metric, a[0], b))  # broadcast query form
    return {"pairs": digest(np.concatenate(pairs)), "broadcast": digest(np.concatenate(broadcast))}


def cosine_parts_inputs():
    rng = np.random.default_rng(3)
    for dim in [1, 3, 4, 5, 17, 128, 768, 1001]:
        for _ in range(20):
            yield rng.standard_normal(dim).astype(np.float32), rng.standard_normal(dim).astype(np.float32)


def _data(rng, n, dim, dup_frac=0.0, clustered=False):
    if clustered:
        c = rng.standard_normal((max(4, int(np.sqrt(n))), dim)).astype(np.float32)
        x = c[rng.integers(0, len(c), n)] + 0.3 * rng.standard_normal((n, dim)).astype(np.float32)
    else:
        x = rng.standard_normal((n, dim)).astype(np.float32)
    if dup_frac > 0:
        k = int(n * dup_frac)
        src = rng.integers(0, n, k)
        dst = rng.integers(0, n, k)
        x[dst] = x[src]
    return np.ascontiguousarray(x, dtype=np.float32)


CONFIGS = [
    # dims, m, efC, efS, n, dup_frac, clustered
    (3, 3, 16, 64, 200, 0.3, False),
    (8, 4, 10, 16, 600, 0.2, False),
    (16, 8, 40, 32, 1500, 0.0, True),
    (33, 5, 20, 64, 800, 0.1, True),
    (128, 16, 64, 64, 1200, 0.0, True),
]


def cfg_id(cfg):
    return f"d{cfg[0]}m{cfg[1]}n{cfg[4]}"


def build_and_search_outputs(oracle_mod, which, metric, cfg):
    dims, m, efc, efs, n, dup, clustered = cfg
    rng = np.random.default_rng(hash((dims, m, n)) % (2**32))
    x = _data(rng, n, dims, dup, clustered)
    if metric == "cosine":
        x += 0.01  # avoid exact zero vectors (NaN distance in the reference, distfunc.c:144)
    q = _data(rng, 50, dims, 0.0, clustered)
    q[:10] = x[:10]  # exact hits
    idx = oracle_mod.FlatIndex(which, dims, m, efc, efs, metric, capacity=n)
    idx.build(x)
    out = {"links": digest(idx.links())}
    for ef in (1, 5, efs):
        r = idx.search_many(q, ef, nthreads=1, want_counters=True)
        out[f"ef{ef}"] = digest(np.concatenate([r["n"].view(np.uint8).ravel(), r["labels"].view(np.uint8).ravel(),
                                                r["counters"].view(np.uint8).ravel()]))  # counters: identical traversal work
    # deleted labels are post-filtered identically
    for i in range(0, n, 3):
        idx.mark_deleted(i)
    r = idx.search_many(q, efs)
    out["deleted"] = digest(np.concatenate([r["n"].view(np.uint8).ravel(), r["labels"].view(np.uint8).ravel()]))
    idx.close()
    return out


def _same(got, want):
    assert got.keys() == want.keys()
    assert [k for k in got if got[k] != want[k]] == []


@pytest.mark.parametrize("metric", METRICS)
def test_distance_bits_all_dims(oracle_mod, metric):
    _same(distance_outputs(oracle_mod, "port", metric), GOLD["dist"][metric])


def test_cosine_parts_recompose(oracle_mod):
    """|b|^2 cached per node + dot recomposes to the exact reference cosine distance."""
    import ctypes as C
    lib = oracle_mod.load("port")
    got = np.array([lib.oracle_cosine_from_parts(a.ctypes.data_as(C.POINTER(C.c_float)), b.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0])
                    for a, b in cosine_parts_inputs()], np.float32)
    assert digest(got) == GOLD["cosine_parts"]


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("cfg", CONFIGS, ids=[cfg_id(c) for c in CONFIGS])
def test_build_and_search_identical(oracle_mod, metric, cfg):
    _same(build_and_search_outputs(oracle_mod, "port", metric, cfg), GOLD["build_search"][f"{metric}.{cfg_id(cfg)}"])
