"""One 'backend' of tests/test_sidecar_dist.py: a separate process with its own connection to the sidecar that evaluates the
SQL distance operators one pair per call, as a Postgres backend does for `val <op> q` in a target list or a WHERE clause
(one hnsw_dist_func per row, embedding.c:1022-1062).  Usage:
    python sidecar_dist_backend.py SHM CALLS.npz OUT.json [REL_KEY DIMS M EFC EFS METRIC EF K]
CALLS.npz holds metric[n], dim[n], a[n, D], b[n, D] (pair i is a[i, :dim[i]], b[i, :dim[i]]).  With the relation arguments
it also holds q[n, DIMS], and call i is one hnsw_search (efSearch EF), one pgemb_client_scan_topk (LIMIT K) and then the
distance of pair i, interleaved.
Output: {"dist": [fp32 bits...], "search": [label lists...], "scan": [{"labels": [...], "dists": [fp32 bits...]}...]}."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

METRIC_NAMES = ("l2", "cosine", "manhattan")


def main():
    shm, calls, out = sys.argv[1:4]
    from pg_embedding_b200 import sidecar
    sidecar.connect(shm)
    c = np.load(calls)
    idx = None
    if len(sys.argv) > 4:
        rel_key, dims, m, efc, efs, metric, ef, k = sys.argv[4:12]
        idx = sidecar.RemoteIndex(int(rel_key), int(dims), int(m), int(efc), int(efs), metric, capacity=1)  # attach = look the mirror up
    # start line: all backends of a test begin together, so that their calls really are concurrent
    open(out + ".ready", "w").close()
    go = os.path.join(os.path.dirname(out), "go")
    deadline = time.time() + 120
    while not os.path.exists(go) and time.time() < deadline:
        time.sleep(0.002)
    res = {"dist": [], "search": [], "scan": []}
    for i in range(c["metric"].size):
        if idx is not None:
            res["search"].append(idx.search(c["q"][i], int(ef)).tolist())
            r = idx.scan_topk(c["q"][i], int(k))
            res["scan"].append({"labels": r["labels"][: r["n"]].tolist(), "dists": r["dists"][: r["n"]].view(np.uint32).tolist()})
        d = int(c["dim"][i])
        res["dist"].append(int(sidecar.dist(METRIC_NAMES[int(c["metric"][i])], c["a"][i, :d], c["b"][i, :d]).view(np.uint32)))
    json.dump(res, open(out, "w"))


if __name__ == "__main__":
    main()
