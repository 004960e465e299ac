"""One 'backend' of tests/test_sidecar_scan_ops.py: a separate process with its own connection to the sidecar that runs
`ORDER BY val <op> q LIMIT k` without the index, one pgemb_client_scan_topk_op call per query (OP = l2 / cosine / manhattan),
or one pgemb_client_scan_topk call per query, which takes the relation's own operator (OP = own).  Usage:
    python sidecar_scan_op_backend.py SHM REL_KEY DIMS M EFC EFS METRIC OP K QUERIES.npy OUT.json
Output: a list of {"labels": [...], "dists": [fp32 bits...]}."""
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
        r = idx.scan_topk(v, int(k), metric=None if op == "own" else op)
        res.append({"labels": r["labels"][: r["n"]].tolist(), "dists": r["dists"][: r["n"]].view(np.uint32).tolist()})
    json.dump(res, open(out, "w"))


if __name__ == "__main__":
    main()
