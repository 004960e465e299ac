"""One 'backend' of tests/test_sidecar_scan.py: a separate process with its own connection to the sidecar that issues one
query per call, like a Postgres backend running `ORDER BY val <op> q LIMIT k` without the index (OP = scan, one
pgemb_client_scan_topk per query) or through it (OP = search, one hnsw_search per query, embedding.c:317).  Usage:
    python sidecar_scan_backend.py SHM REL_KEY DIMS M EFC EFS METRIC OP K_OR_EF QUERIES.npy OUT.json
Output: for `scan` a list of {"labels": [...], "dists": [fp32 bits...]}, for `search` a list of label lists."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    shm, rel_key, dims, m, efc, efs, metric, op, k, qpath, out = sys.argv[1:12]
    from pg_embedding_b200 import sidecar
    sidecar.connect(shm)
    idx = sidecar.RemoteIndex(int(rel_key), int(dims), int(m), int(efc), int(efs), metric, capacity=1)  # attach = look the mirror up
    q = np.load(qpath)
    # start line: all backends of a test begin together, so that their calls really are concurrent
    open(out + ".ready", "w").close()
    go = os.path.join(os.path.dirname(out), "go")
    deadline = time.time() + 120
    while not os.path.exists(go) and time.time() < deadline:
        time.sleep(0.002)
    res = []
    for v in q:
        if op == "scan":
            r = idx.scan_topk(v, int(k))
            res.append({"labels": r["labels"][: r["n"]].tolist(), "dists": r["dists"][: r["n"]].view(np.uint32).tolist()})
        else:
            res.append(idx.search(v, int(k)).tolist())
    json.dump(res, open(out, "w"))


if __name__ == "__main__":
    main()
