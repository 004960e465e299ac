#!/usr/bin/env python
"""Generate golden fixtures from the UNMODIFIED compiled reference (oracle/_ref/libpgemb_ref.so = the reference's
hnswalg.cpp + distfunc.c built in place by oracle/Makefile, on the flat-memory host).  Needs the reference sources:

    python tests/golden/gen_ref_fixtures.py

Writes tests/golden/ref_fixtures.npz: seeded inputs, the reference's link lists after a sequential build, its
hnsw_search results and its hnsw_dist_func outputs (raw fp32 bits).  tests/test_golden_fixtures.py checks the C
restatement (and, on a GPU, the CUDA path) against this file without needing the reference tree.

Writes tests/golden/ref_compare.json: the reference's outputs on the seeded inputs of tests/test_oracle_vs_ref.py (SHA-256
of the raw bytes) and the HnswMetadata field list of its embedding.h (tests/test_abi.py)."""
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import oracle  # noqa: E402
import test_oracle_vs_ref as vs  # noqa: E402

oracle.build("ref")
assert oracle.available("ref"), "needs the reference sources to build oracle/_ref"
out = {}
CASES = [  # name, dims, m, efC, n, metric, tie-heavy?
    ("l2_d8", 8, 4, 16, 300, "l2", False),
    ("cos_d33", 33, 5, 24, 300, "cosine", False),
    ("man_d16", 16, 6, 20, 300, "manhattan", False),
    ("l2_ties_d3", 3, 3, 16, 200, "l2", True),
    ("cos_d768", 768, 8, 32, 160, "cosine", False),
]
for name, dims, m, efc, n, metric, ties in CASES:
    rng = np.random.default_rng(sum(map(ord, name)))
    if ties:
        x = rng.integers(0, 3, size=(n, dims)).astype(np.float32)
        q = rng.integers(0, 3, size=(24, dims)).astype(np.float32)
    else:
        x = rng.standard_normal((n, dims)).astype(np.float32)
        q = rng.standard_normal((24, dims)).astype(np.float32)
    if metric == "cosine":
        x, q = x + 1.0, q + 1.0
    labels = (rng.permutation(n).astype(np.uint64) << np.uint64(20)) | np.uint64(3)
    idx = oracle.FlatIndex("ref", dims, m, efc, 16, metric, capacity=n)
    idx.build(x, labels)
    for i in range(0, n, 7):
        idx.mark_deleted(i)
    res = idx.search_many(q, 16, nthreads=1)
    res5 = idx.search_many(q, 5, nthreads=1)
    out[f"{name}.params"] = np.array([dims, m, efc, n, oracle.METRICS[metric]], dtype=np.int64)
    out[f"{name}.x"], out[f"{name}.q"] = x, q
    out[f"{name}.labels"] = idx.labels()
    out[f"{name}.links"] = idx.links()
    out[f"{name}.search16"], out[f"{name}.n16"] = res["labels"], res["n"]
    out[f"{name}.search5"], out[f"{name}.n5"] = res5["labels"], res5["n"]
    out[f"{name}.dist_bits"] = oracle.dist_many("ref", metric, q[0], x).view(np.uint32)
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_fixtures.npz"), **out)
print("wrote ref_fixtures.npz with", len(out), "arrays")

cmp = {"dist": {m: vs.distance_outputs(oracle, "ref", m) for m in vs.METRICS},
       "cosine_parts": vs.digest(np.array([oracle.dist("ref", "cosine", a, b) for a, b in vs.cosine_parts_inputs()], np.float32)),
       "build_search": {f"{m}.{vs.cfg_id(c)}": vs.build_and_search_outputs(oracle, "ref", m, c) for m in vs.METRICS for c in vs.CONFIGS},
       "metadata_fields": re.findall(r"^\s*(?:size_t|idx_t|dist_func_t)\s+(\w+);", open(os.path.join(oracle.REF_SRC, "embedding.h")).read(), re.M)}
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_compare.json"), "w") as f:
    json.dump(cmp, f, indent=1, sort_keys=True)
    f.write("\n")
print("wrote ref_compare.json")
