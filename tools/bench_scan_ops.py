#!/usr/bin/env python
"""The exact scan under each operator over a mirror of each metric (pgemb_scan_topk_op_device): 1024 queries x 1M rows x 768
dims by default, all 3 x 3 (mirror metric, query metric) pairs in one process.

One JSON line per pair: ms per call (median and min over --steps timed calls, host clock around a call that returns after
its scan has finished), the pgemb_scan_counters deltas of one call, and against the matched pair of the same query metric
(the mirror whose own metric it is): the time ratio and whether the results are the same bytes -- all three mirrors hold the
same rows under the same labels, so they must be.  Every line names the GPU and its power limit, read in the same run.
usage: bench_scan_ops.py [--n 1000000 --dims 768 --nq 1024 --k 64 --steps 5 --warmup 1 --out FILE]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import pg_embedding_b200 as pg  # noqa: E402
from pg_embedding_b200 import _lib  # noqa: E402

METRICS = ("l2", "cosine", "manhattan")


def card():
    """The card's name and power limit (read-only nvidia-smi query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, plim = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit_w": float(plim)}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}


def counters(lib):
    out = (C.c_uint64 * 6)()
    lib.pgemb_scan_counters(out)
    return dict(zip(("tc", "pairs", "rescored", "fallbacks", "overflow", "exact"), list(out)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dims", type=int, default=768)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--k", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    lib = _lib.load()
    if pg.device_count() < 1:
        sys.exit("no CUDA device: this measurement needs the GPU")
    hw = card()
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    # clustered rows (what a filter meets in practice) shifted off the origin, so that cosine is not degenerate
    centres = torch.randn((1000, a.dims), generator=g, device="cuda")
    X = torch.empty((a.n, a.dims), device="cuda")
    for s in range(0, a.n, 1 << 16):
        e = min(a.n, s + (1 << 16))
        c = torch.randint(0, centres.shape[0], (e - s,), generator=g, device="cuda")
        X[s:e] = centres[c] + 0.3 * torch.randn((e - s, a.dims), generator=g, device="cuda") + 0.5
    c = torch.randint(0, centres.shape[0], (a.nq,), generator=g, device="cuda")
    Q = (centres[c] + 0.3 * torch.randn((a.nq, a.dims), generator=g, device="cuda") + 0.5).contiguous()
    stream = torch.cuda.current_stream().cuda_stream
    mirrors = {}
    for m in METRICS:
        idx = pg.HnswIndex(a.dims, 16, 64, 64, m, capacity=a.n)
        _lib.check(lib.pgemb_index_append_device(idx.dev, a.n, X.data_ptr(), None, None, stream))
        mirrors[m] = idx
    torch.cuda.synchronize()
    del X
    lab = torch.empty((a.nq, a.k), dtype=torch.int64, device="cuda")
    dst = torch.empty((a.nq, a.k), dtype=torch.float32, device="cuda")
    cnt = torch.empty((a.nq,), dtype=torch.int32, device="cuda")

    def scan(mirror, metric):
        _lib.check(lib.pgemb_scan_topk_op_device(mirrors[mirror].dev, METRICS.index(metric), a.nq, Q.data_ptr(), a.k, lab.data_ptr(), dst.data_ptr(),
                                                 cnt.data_ptr(), None))

    rows, results = [], {}
    for mirror in METRICS:
        for metric in METRICS:
            c0 = counters(lib)
            scan(mirror, metric)      # the first call of a pair: a mirror without row norms computes them here
            first = {k: v - c0[k] for k, v in counters(lib).items()}
            results[(mirror, metric)] = (lab.cpu().numpy().tobytes(), dst.cpu().numpy().tobytes(), cnt.cpu().numpy().tobytes())
            for _ in range(max(0, a.warmup - 1)):
                scan(mirror, metric)
            c0 = counters(lib)
            ts = []
            for _ in range(a.steps):
                t = time.perf_counter()
                scan(mirror, metric)
                ts.append(1e3 * (time.perf_counter() - t))
            per_call = {k: (v - c0[k]) / a.steps for k, v in counters(lib).items()}
            rows.append(dict(mirror=mirror, query=metric, ms_median=float(np.median(ts)), ms_min=float(np.min(ts)), counters_first_call=first,
                             counters_per_call=per_call))
    matched = {r["query"]: r for r in rows if r["mirror"] == r["query"]}
    lines = []
    for r in rows:
        r["vs_matched"] = {"ratio_median": r["ms_median"] / matched[r["query"]]["ms_median"],
                           "identical_results": results[(r["mirror"], r["query"])] == results[(r["query"], r["query"])]}
        r.update(hw, n=a.n, dims=a.dims, nq=a.nq, k=a.k, steps=a.steps)
        lines.append(json.dumps(r))
    for line in lines:
        print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")
    for idx in mirrors.values():
        idx.close()
    if not all(json.loads(line)["vs_matched"]["identical_results"] for line in lines):
        sys.exit("a mismatched pair's results differ from the matched pair's")


if __name__ == "__main__":
    main()
