"""Known-answer tests: the C restatement (`port`) against the results the reference's own pg_regress suite pins
(tests/golden/kat_regress.json, transcribed from the reference's test/expected/*.out)."""
import json
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(__file__), "golden", "kat_regress.json")
CASES = json.load(open(GOLD))["cases"]


def tid_label(blk: int, pos: int, flags: int = 0) -> int:
    """HnswLabel (embedding.c:50-56): {BlockIdData{bi_hi,bi_lo}, ip_posid, flags} as a little-endian u64."""
    return (blk >> 16) | ((blk & 0xFFFF) << 16) | (pos << 32) | (flags << 48)


def run_case(oracle_mod, which, case, metric):
    o = case["options"]
    idx = oracle_mod.FlatIndex(which, o["dims"], o["m"], o["efconstruction"], o["efsearch"], metric, capacity=64)
    by_label = {}
    for r in case.get("rows_before_truncate", []):
        idx.add(np.array(r["val"], np.float32), tid_label(*r["tid"]))
    if "rows_before_truncate" in case:
        idx.truncate()  # TRUNCATE gives the index a fresh, empty relation (gh-3)
    for r in case["rows"]:
        lab = tid_label(*r["tid"])
        idx.add(np.array(r["val"], np.float32), lab)
        by_label[lab] = r
    if "delete_all_then_insert" in case:
        for i in range(len(idx)):
            idx.mark_deleted(i)  # ambulkdelete after `delete from t; vacuum t`
        by_label = {}
        for r in case["delete_all_then_insert"]:
            lab = tid_label(*r["tid"])
            idx.add(np.array(r["val"], np.float32), lab)
            by_label[lab] = r
    labels = idx.search(np.array(case["query"], np.float32))
    return [by_label[int(l)] for l in labels], idx


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
@pytest.mark.parametrize("which", ["port"])
def test_kat(oracle_mod, which, case):
    metrics = list(case.get("expected", case.get("expected_tids")).keys())
    for metric in metrics:
        rows, idx = run_case(oracle_mod, which, case, metric)
        if "expected" in case:
            assert [r["val"] for r in rows] == case["expected"][metric], (which, metric)
        if "expected_tids" in case:
            assert [r["tid"] for r in rows] == case["expected_tids"][metric], (which, metric)
        if "expected_distances" in case:
            q = np.array(case["query"], np.float32)
            got = [float(oracle_mod.dist(which, metric, q, np.array(r["val"], np.float32))) for r in rows]
            np.testing.assert_allclose(got, case["expected_distances"][metric], rtol=0, atol=5e-7)


def test_kat_seqscan_equals_index(oracle_mod):
    """knn.out:63-91: the seq-scan (exact) order equals the index order on the KAT data, all 3 metrics."""
    case = CASES[0]
    q = np.array(case["query"], np.float32)
    for metric in ("l2", "cosine", "manhattan"):
        vals = [np.array(r["val"], np.float32) for r in case["rows"]]
        labs = [tid_label(*r["tid"]) for r in case["rows"]]
        d = [float(oracle_mod.dist("port", metric, q, v)) for v in vals]
        order = sorted(range(len(vals)), key=lambda i: (d[i], labs[i]))
        assert [case["rows"][i]["val"] for i in order] == case["expected"][metric]
